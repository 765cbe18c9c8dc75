// emu_parse.cpp -- the MatcherParser stage (dm_kernels_parse.cuh) on the CPU emulator.  TEST INFRASTRUCTURE ONLY:
// tests/test_matcher_parser.py builds it into its own library under tests/emu/_build/; never part of libdmdetect.so.
//
// It is emu.cpp (every emu_* entry point, the emulated handle, the launch helpers) plus the dm_parse_logs sequence: the
// framing of dm_host.h, the unwrap kernels without the text copy, the size pass, the scan and the write pass, the
// grid-stride kernels on 2 CTAs so that batches of more than 128 records take their stride loops, every scratch array
// starting out hostile.
#include "emu.cpp"

#include "dm_kernels_parse.cuh"

// As dm_set_parser_format + dm_parse_logs, on the format of emu_set_format (call emu_set_monitors first, with no
// monitors).  out: out_cap bytes.  Returns 0; -1 for a framing error, -2 when dm_parse_fmt_build refuses the strings
// (*why), -4 when the output exceeds out_cap (*out_len then tells how large).
extern "C" int emu_parse_logs(EmuHandle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* lens,
                              const uint32_t* capture_order, const uint8_t* msg, uint64_t nbytes, int delimited,
                              int64_t first_id, int64_t now, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                              uint64_t* n_records, uint64_t* n_emitted, const char** why) {
    static DmParseFmt P;
    static DmFormat pfmt;
    *why = dm_parse_fmt_build(h->fmt, n_strings, strings, lens, capture_order, &P);
    if (*why) return -2;
    dm_parse_efmt_build(h->fmt, &pfmt);
    const DmFrames fr = dm_frame_records(msg, nbytes, delimited != 0);
    if (fr.error) return -1;
    const uint32_t n = (uint32_t)fr.off.size();
    std::vector<uint8_t> buf(nbytes + 64, 0x0A);                     // hostile slack: '\n' bytes
    memcpy(buf.data(), msg, nbytes);
    std::vector<uint8_t> nbuf(nbytes + 256, 0xA5);
    uint32_t per_cta;
    const uint32_t n_chunks = dm_logs_plan(n, 2, &per_cta);
    std::vector<uint32_t> text_off(n + 1, 0xDEADBEEFu), text_len(n + 1, 0xDEADBEEFu), rec_line(n + 1, 0xDEADBEEFu);
    std::vector<uint32_t> line_src(n + 1), line_dst(n + 1), line_rec(n + 1);
    std::vector<unsigned long long> loc(n + 1), chunk(n_chunks + 1);
    DmLogsHeader lh;
    memset(&lh, 0, sizeof(lh));
    DmLogsArgs la;
    la.buf = buf.data(); la.rec_off = fr.off.data(); la.rec_len = fr.len.data(); la.n_records = n; la.n_train_records = 0;
    la.per_cta = per_cta; la.n_chunks = n_chunks; la.text_off = text_off.data(); la.text_len = text_len.data();
    la.loc = loc.data(); la.chunk = chunk.data(); la.rec_line = rec_line.data(); la.line_src = line_src.data();
    la.line_dst = line_dst.data(); la.line_rec = line_rec.data(); la.out = nullptr; la.out_cap = 0; la.lhdr = &lh;
    std::vector<unsigned long long> size(n + 1, 0xDEADBEEFull), tiles(n / DMA_TILE + 2, 0xDEADBEEFull);
    unsigned long long total = 0;
    std::vector<uint8_t> dout(out_cap + 1, 0xEE);
    DmParseArgs a;
    a.pf = &P; a.pfmt = &pfmt; a.buf = buf.data(); a.nbuf = nbuf.data(); a.n_records = n;
    a.rec_off = fr.off.data(); a.rec_len = fr.len.data(); a.text_off = text_off.data(); a.text_len = text_len.data();
    a.rank = rec_line.data(); a.size = size.data(); a.first_id = first_id; a.now = now;
    a.out = dout.data(); a.out_cap = out_cap; a.total = &total;
    const bool norm = dm_format_norm(h->fmt);
    auto pass = [&](bool write) {
        g_emu_dyn_smem.assign((size_t)2 * pfmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
        const DmParseKernel k = dm_parse_kernel(norm, write);
        emu_launch_grid(2, DM_FMTL_THREADS, [&] { k(a); });
    };
    if (n) {
        emu_launch_grid(n_chunks, DML_THREADS, [&] { dm_k_logs_walk(la); });
        emu_launch_grid(1, DML_THREADS, [&] { dm_k_logs_scan(la); });
        emu_launch_grid(2, DML_THREADS, [&] { dm_k_logs_compact(la); });
        pass(false);
        const uint32_t nt = (uint32_t)std::max<uint64_t>(1, (n + DMA_TILE - 1) / DMA_TILE);
        emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_tiles<unsigned long long>(size.data(), n, tiles.data()); });
        emu_launch(DMA_THREADS, [&] { dm_k_alert_scan_top<unsigned long long>(tiles.data(), nt, &total); });
        emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_apply<unsigned long long>(size.data(), n, tiles.data()); });
    }
    *out_len = total;
    *n_records = n;
    *n_emitted = lh.n_lines;
    if (total > out_cap) return -4;
    if (total) pass(true);
    memcpy(out, dout.data(), total);
    return 0;
}
