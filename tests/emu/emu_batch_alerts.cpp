// emu_batch_alerts.cpp -- the DetectorSchema encoder of LogSchema and ParserSchema batches (dm_kernels_alerts.cuh) on
// the CPU emulator.  TEST INFRASTRUCTURE ONLY: tests/test_emu_record_alerts.py builds it into its own library under
// tests/emu/_build/; never part of libdmdetect.so.
//
// It is emu.cpp (every emu_* entry point, the emulated handle, the launch helpers) plus the entry points of this
// input: the whole dm_process_logs sequence, and the encoder passes after it or after dm_process_records, with the same
// hostile scratch and 2-CTA grid-stride conventions as emu_encode_alerts.
#include "emu.cpp"

#include <map>

// What dm_process_logs leaves on the device for dm_encode_alerts, per emulated handle: the message, the unwrap arrays,
// the compacted texts and the per-record scores.
struct EmuLogs {
    std::vector<uint8_t> msg, text;
    std::vector<uint32_t> rec_off, rec_len, rec_line, line_dst;
    std::vector<float> rscores;
    uint64_t total = 0;
};
static std::map<const EmuHandle*, EmuLogs> g_emu_logs;

// the anomaly list's capacity (dm_handle::anomaly_cap; 65536 from emu_create)
extern "C" void emu_set_anomaly_cap(EmuHandle* h, uint32_t cap) { h->anoms.assign(cap ? cap : 1, dm_anomaly_t{}); }

// emu_destroy, also forgetting the handle's last LogSchema batch
extern "C" void emu_batch_destroy(EmuHandle* h) {
    g_emu_logs.erase(h);
    emu_destroy(h);
}

// The encoder passes of dm_encode_alerts on the emulator, for the arguments in `a` (src, pay ... set by the caller):
// the grid-stride kernels run on 2 CTAs, so that batches of more than 512 (log_format: 128) anomalous records take their
// stride loops; every scratch array, the R-norm scratch included, starts out hostile.  buf / nbytes: the text the
// key=value and log_format passes read (hostile slack is added), fmt: log_format mode.
static int emu_alert_passes(EmuHandle* h, DmAlertArgs a, bool fmt, const uint8_t* msg, uint64_t nbytes, uint32_t entries,
                            uint64_t n_lines, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    const bool records = a.src == DMA_RECORDS;
    std::vector<uint8_t> buf(nbytes + 64, 'x');                      // hostile slack: no record may reach into it
    if (nbytes) memcpy(buf.data(), msg, nbytes);
    std::vector<uint32_t> rank(n_lines + 1, 0), rec_line(entries + 1, 0xDEADBEEFu), rec_mask(entries + 1, 0);
    std::vector<unsigned long long> rec_off(entries + 1, 0xDEADBEEFull), size(entries + 1, 0xDEADBEEFull);
    std::vector<unsigned long long> tiles(std::max<uint64_t>(n_lines, entries) / DMA_TILE + 2, 0xDEADBEEFull);
    std::vector<uint8_t> dout(out_cap + 1, 0xEE);
    DmAlertHeader ah;
    memset(&ah, 0, sizeof(ah));
    a.fmt = &h->afmt; a.buf = buf.data(); a.nbytes = nbytes; a.anoms = h->anoms.data();
    a.n_entries = entries; a.n_lines = n_lines; a.rank = rank.data(); a.rec_line = rec_line.data(); a.rec_mask = rec_mask.data();
    a.rec_off = rec_off.data(); a.size = size.data(); a.ahdr = &ah; a.out = dout.data(); a.out_cap = out_cap;
    static DmFormat efmt;
    dm_alert_efmt_build(h->fmt, h->afmt.time_cap, &efmt);
    std::vector<uint8_t> nbuf(nbytes + 256, 0xA5);
    a.efmt = &efmt; a.nbuf = nbuf.data();
    const bool norm = dm_format_norm(h->fmt);
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
    if (records) emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_mark_records(a); });
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_mark(a); });
    scan(rank.data(), n_lines, &ah.n_alerts);
    if (records) emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_gather_records(a); });
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_gather(a); });
    if (records) emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_records<false>(a); });
    else if (fmt) fmt_pass(false);
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_size(a); });
    scan(size.data(), (uint64_t)entries, &ah.total);
    if (records) emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_records<true>(a); });
    else if (fmt) fmt_pass(true);
    else emu_launch_grid(2, DMA_THREADS, [&] { dm_k_alert_write(a); });
    *n_alerts = ah.n_alerts;
    *out_len = ah.total;
    if (ah.declined || ah.total > out_cap) { *declined = 1; return 0; }
    memcpy(out, dout.data(), ah.total);
    return 0;
}

// ---------------------------------------------------------------------------------------------- LogSchema batches
// As dm_process_logs: the framing, the four unwrap kernels (walk grid capped at 2 CTAs), the line path of `variant` (0
// stream, 1 stream with the chained re-check, 2 lanes, 3 log_format) on the compacted texts, then dm_k_logs_scatter on 2
// CTAs.  flags / scores: per record (cap entries).  The handle keeps what dm_encode_alerts reads (emu_encode_log_alerts).
// Returns 0, -1 for a framing error, -4 when the records exceed cap, or the line path's error.
extern "C" int emu_process_logs(EmuHandle* h, int variant, const uint8_t* msg, uint64_t nbytes, int delimited, uint32_t n_train,
                                uint8_t* flags, float* scores, uint64_t cap, uint64_t* n_records, uint64_t* n_malformed,
                                uint64_t* n_anoms) {
    DmFrames fr;
    if (delimited) {
        fr = dm_frame_split(msg, nbytes);
        if (fr.error) return -1;
    } else {
        fr.off.push_back(0);
        fr.len.push_back((uint32_t)nbytes);
    }
    const uint32_t n = (uint32_t)fr.off.size();
    if (n > cap) return -4;
    EmuLogs& L = g_emu_logs[h];
    L.msg.assign(nbytes + 64, 0x0A);                                 // hostile slack: '\n' bytes
    memcpy(L.msg.data(), msg, nbytes);
    L.rec_off = fr.off; L.rec_len = fr.len;
    L.rec_line.assign(n + 1, 0xDEADBEEFu); L.line_dst.assign(n + 1, 0xDEADBEEFu);
    L.rscores.assign(n + 1, -1.0f);
    const uint64_t out_cap = (nbytes + 1 + DML_SLACK + 15) & ~15ull;
    L.text.assign(out_cap, 0xEE);
    uint32_t per_cta;
    const uint32_t n_chunks = dm_logs_plan(n, 2, &per_cta);
    std::vector<uint32_t> text_off(n + 1), text_len(n + 1), line_src(n + 1), line_rec(n + 1, 0xDEADBEEFu);
    std::vector<unsigned long long> loc(n + 1), chunk(n_chunks + 1);
    std::vector<uint8_t> rflags(n + 1, 7);
    DmLogsHeader lh;
    memset(&lh, 0, sizeof(lh));
    DmLogsArgs a;
    a.buf = L.msg.data(); a.rec_off = L.rec_off.data(); a.rec_len = L.rec_len.data(); a.n_records = n; a.n_train_records = n_train;
    a.per_cta = per_cta; a.n_chunks = n_chunks; a.text_off = text_off.data(); a.text_len = text_len.data();
    a.loc = loc.data(); a.chunk = chunk.data(); a.rec_line = L.rec_line.data(); a.line_src = line_src.data();
    a.line_dst = L.line_dst.data(); a.line_rec = line_rec.data(); a.out = L.text.data(); a.out_cap = out_cap; a.lhdr = &lh;
    if (n) {
        emu_launch_grid(n_chunks, DML_THREADS, [&] { dm_k_logs_walk(a); });
        emu_launch_grid(1, DML_THREADS, [&] { dm_k_logs_scan(a); });
        emu_launch_grid(2, DML_THREADS, [&] { dm_k_logs_compact(a); });
        emu_launch_grid(2, DML_THREADS, [&] { dm_k_logs_copy(a); });
    }
    L.total = lh.total_bytes;
    std::vector<uint8_t> lflags(lh.n_lines + 2, 7);
    std::vector<float> lscores(lh.n_lines + 2, -1.0f);
    if (lh.n_lines) {
        uint64_t nl = 0, na = 0;
        uint32_t err = 0;
        int rc;
        if (variant <= 1) rc = emu_stream_run(h, variant == 1, L.text.data(), lh.total_bytes, lh.n_train, lflags.data(), lscores.data(),
                                             lh.n_lines + 2, &nl, &na, &err);
        else if (variant == 2) rc = emu_process_lanes(h, L.text.data(), lh.total_bytes, lh.n_train, lflags.data(), lscores.data(),
                                                      lh.n_lines + 2, &nl, &na, &err);
        else rc = emu_process_format(h, L.text.data(), lh.total_bytes, lh.n_train, lflags.data(), lscores.data(), lh.n_lines + 2,
                                     &nl, &na, &err);
        if (rc != 0) return rc;
        if (err || nl != lh.n_lines) return -5;
    } else {
        memset(&h->hdr, 0, sizeof(h->hdr));
    }
    unsigned long long stats[DM_STATS_WORDS] = {0};
    emu_launch_grid(2, DML_THREADS, [&] {
        dm_k_logs_scatter(a, lflags.data(), lscores.data(), rflags.data(), L.rscores.data(), h->anoms.data(),
                          (uint32_t)h->anoms.size(), &h->hdr, stats, nbytes);
    });
    for (int i = 0; i < DM_STATS_WORDS; ++i) h->stats[i] += stats[i];
    memcpy(flags, rflags.data(), n);
    memcpy(scores, L.rscores.data(), (uint64_t)n * 4);
    *n_records = n;
    *n_malformed = n - lh.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    return 0;
}

// As dm_encode_alerts after dm_process_logs: the batch of the last emu_process_logs; fmt: it ran in log_format mode.
extern "C" int emu_encode_log_alerts(EmuHandle* h, int fmt, int64_t first_alert_id, int64_t now, uint8_t* out, uint64_t out_cap,
                                     uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    const auto it = g_emu_logs.find(h);
    if (!h->afmt_set || it == g_emu_logs.end()) return -6;
    *out_len = 0; *n_alerts = 0; *declined = 0;
    const EmuLogs& L = it->second;
    const uint32_t entries = std::min<uint32_t>(h->hdr.anomaly_list_count, (uint32_t)h->anoms.size());
    const uint64_t n_lines = h->hdr.n_lines;
    if (entries == 0 || n_lines == 0) return 0;
    DmAlertArgs a;
    a.scores = L.rscores.data(); a.first_log_id = 0; a.first_alert_id = first_alert_id; a.now = now;
    a.src = DMA_LOGS; a.pay = L.msg.data(); a.pay_off = L.rec_off.data(); a.pay_len = L.rec_len.data();
    a.log_line = L.rec_line.data(); a.log_dst = L.line_dst.data();
    return emu_alert_passes(h, a, fmt != 0, L.text.data(), L.total, entries, n_lines, out, out_cap, out_len, n_alerts, declined);
}

// As dm_encode_alerts after dm_process_records: msg is the batch of the last emu_process_records and flags / scores /
// masks its outputs.  A batch with more anomalous records than the anomaly list holds (emu_set_anomaly_cap) declines.
extern "C" int emu_encode_record_alerts(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, const uint8_t* flags,
                                        const float* scores, const uint32_t* masks, int64_t first_alert_id, int64_t now,
                                        uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    if (!h->afmt_set) return -6;
    *out_len = 0; *n_alerts = 0; *declined = 0;
    const DmFrames fr = dm_frame_split(msg, nbytes);
    if (fr.error) return -1;
    const uint64_t n_lines = fr.off.size(), n_flagged = h->hdr.n_anomalies;
    if (n_flagged == 0 || n_lines == 0) return 0;
    if (n_flagged > h->anoms.size()) { *n_alerts = n_flagged; *declined = 1; return 0; }
    std::vector<uint8_t> pay(nbytes + 64, 0x0A);                     // hostile slack
    memcpy(pay.data(), msg, nbytes);
    DmAlertArgs a;
    a.scores = scores; a.first_log_id = 0; a.first_alert_id = first_alert_id; a.now = now;
    a.src = DMA_RECORDS; a.pay = pay.data(); a.pay_off = fr.off.data(); a.pay_len = fr.len.data();
    a.flags = flags; a.masks = masks; a.mons = &h->mons;
    return emu_alert_passes(h, a, false, nullptr, 0, (uint32_t)n_flagged, n_lines, out, out_cap, out_len, n_alerts, declined);
}

// The device's Time conversion of the UTF-8 of a str (a ParserSchema Time): 1 and *ts = int(float(s)), or `now` where
// float() must raise ValueError; 0 (declined) otherwise.
extern "C" int emu_alert_time_str(const uint8_t* s, uint32_t n, long long now, long long* ts) {
    return dma_time(s, n, now, ts, true) ? 1 : 0;
}
