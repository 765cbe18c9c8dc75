// emu_alerts.cpp -- the emulator of emu_tile.cpp and the format emulator (emu_format_combo.cpp) running the
// DetectorSchema encoder kernels (dm_kernels_alerts.cuh) on the batch the last emu_process_{stream,stream_chain,lanes,
// format,format_combo} call detected, launched as dm_encode_alerts launches them.  TEST INFRASTRUCTURE ONLY: built by
// tests/test_emu_alerts.py into tests/emu/_build/; never part of libdmdetect.so.  It includes emu_format_combo.cpp (and
// so emu_tile.cpp) whole, so this library exports every emu_* function of both as well.
#include "emu_format_combo.cpp"

#include <type_traits>

#include "dm_kernels_alerts.cuh"

static DmAlertFmt g_afmt;
static bool g_afmt_set = false;

// mirrors dm_set_alert_format (the monitors' keys are those of emu_create); nullptr or the reason it refuses
extern "C" const char* emu_set_alert_format(EmuHandle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* lens,
                                            const uint32_t* bits_off, const uint32_t* bits, uint32_t n_combos,
                                            const uint32_t* combo_off, const uint32_t* members, uint32_t time_cap) {
    const char* why = dm_alert_fmt_build(h->keys, n_strings, strings, lens, bits_off, bits, n_combos, combo_off, members,
                                         time_cap, &g_afmt);
    g_afmt_set = why == nullptr;
    return why;
}

// Mirrors dm_encode_alerts on the last batch: msg / scores are that batch's message and scores (the emulated detect
// functions do not keep them); fmt: the batch was detected in log_format mode (emu_set_format's format).  The
// grid-stride kernels run on 2 CTAs, so that batches of more than 512 (log_format: 128) anomaly entries take their
// stride loops; every scratch array, the R-norm scratch included, starts out hostile.  Returns 0, or -6 without an alert
// format.
extern "C" int emu_encode_alerts(EmuHandle* h, int fmt, const uint8_t* msg, uint64_t nbytes, const float* scores,
                                 uint64_t first_log_id, int64_t first_alert_id, int64_t now, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    if (!g_afmt_set) return -6;
    *out_len = 0; *n_alerts = 0; *declined = 0;
    const uint32_t entries = std::min<uint32_t>(h->hdr.anomaly_list_count, (uint32_t)h->anoms.size());
    const uint64_t n_lines = h->hdr.n_lines;
    if (entries == 0 || n_lines == 0) return 0;
    std::vector<uint8_t> buf(nbytes + 64, 'x');                      // hostile slack: no record may reach into it
    memcpy(buf.data(), msg, nbytes);
    std::vector<uint32_t> rank(n_lines + 1, 0), rec_line(entries + 1, 0xDEADBEEFu), rec_mask(entries + 1, 0);
    std::vector<unsigned long long> rec_off(entries + 1, 0xDEADBEEFull), size(entries + 1, 0xDEADBEEFull);
    std::vector<unsigned long long> tiles(std::max<uint64_t>(n_lines, entries) / DMA_TILE + 2, 0xDEADBEEFull);
    std::vector<uint8_t> dout(out_cap + 1, 0xEE);
    DmAlertHeader ah;
    memset(&ah, 0, sizeof(ah));
    DmAlertArgs a;
    a.fmt = &g_afmt; a.buf = buf.data(); a.nbytes = nbytes; a.scores = scores; a.anoms = h->anoms.data();
    a.n_entries = entries; a.n_lines = n_lines; a.rank = rank.data(); a.rec_line = rec_line.data(); a.rec_mask = rec_mask.data();
    a.rec_off = rec_off.data(); a.size = size.data(); a.ahdr = &ah; a.first_log_id = first_log_id;
    a.first_alert_id = first_alert_id; a.now = now; a.out = dout.data(); a.out_cap = out_cap;
    static DmFormat efmt;
    dm_alert_efmt_build(g_fmt, g_afmt.time_cap, &efmt);
    std::vector<uint8_t> nbuf(nbytes + 256, 0xA5);
    a.efmt = &efmt; a.nbuf = nbuf.data();
    const bool norm = g_fmt.norm_flags != 0 && g_fmt.n_chains > 1;
    auto fmt_pass = [&](bool write) {
        g_emu_dyn_smem.assign((size_t)2 * efmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
        if (norm && write) emu_launch_grid(2, DM_FMTL_THREADS, [&] { dm_k_alert_format<true, true>(a); });
        else if (norm) emu_launch_grid(2, DM_FMTL_THREADS, [&] { dm_k_alert_format<true, false>(a); });
        else if (write) emu_launch_grid(2, DM_FMTL_THREADS, [&] { dm_k_alert_format<false, true>(a); });
        else emu_launch_grid(2, DM_FMTL_THREADS, [&] { dm_k_alert_format<false, false>(a); });
    };
    auto scan = [&](auto* d, uint64_t n, auto* total) {
        using T = std::remove_pointer_t<decltype(d)>;
        T* ts = (T*)tiles.data();
        const uint32_t nt = (uint32_t)std::max<uint64_t>(1, (n + DMA_TILE - 1) / DMA_TILE);
        emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_tiles<T>(d, n, ts); });
        emu_launch(DMA_THREADS, [&] { dm_k_alert_scan_top<T>(ts, nt, total); });
        emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_apply<T>(d, n, ts); });
    };
    emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_mark(a); });
    scan(rank.data(), n_lines, &ah.n_alerts);
    emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_gather(a); });
    if (fmt) fmt_pass(false);
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_size(a); });
    scan(size.data(), (uint64_t)entries, &ah.total);
    if (fmt) fmt_pass(true);
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_write(a); });
    *n_alerts = ah.n_alerts;
    *out_len = ah.total;
    if (ah.declined || ah.total > out_cap) { *declined = 1; return 0; }
    memcpy(out, dout.data(), ah.total);
    return 0;
}

// The device's UTF-8 replacement of one value (bytes written to out, at most 3 per input byte); its length.
extern "C" uint32_t emu_utf8_replace(const uint8_t* s, uint32_t n, uint8_t* out) {
    DmaOut w{out, 0};
    dma_utf8_replace(w, s, n);
    return (uint32_t)w.n;
}

// The device's Time conversion: 1 and *ts = int(float(s)), or `now` where float() must raise ValueError; 0 (declined)
// otherwise.
extern "C" int emu_alert_time(const uint8_t* s, uint32_t n, long long now, long long* ts) { return dma_time(s, n, now, ts) ? 1 : 0; }
