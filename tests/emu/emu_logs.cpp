// emu_logs.cpp -- the emulator of emu_tile.cpp running the LogSchema unwrap kernels (dm_kernels_logs.cuh): walk, scan,
// compact and copy, launched as dm_process_logs launches them.  TEST INFRASTRUCTURE ONLY: built by
// tests/test_logschema.py into tests/emu/_build/; never part of libdmdetect.so.
#include "emu_tile.cpp"
#include "dm_kernels_logs.cuh"

// Frames the message as dm_process_logs does, then runs the four unwrap kernels with the walk grid capped at
// `walk_ctas` CTAs (so that a CTA walks several tiles of records) and the copy on `copy_ctas` CTAs (so that its threads
// take the grid-stride loop).  The message is followed by hostile bytes, the output buffer is pre-filled with 0xEE.
// Outputs: out (the compacted texts and the slack), rec_line / line_rec / line_dst, hdr = {total_bytes, n_lines,
// n_train, bound}.  Returns the record count, or -1 for a framing error.
extern "C" int64_t emu_logs_unwrap(const uint8_t* msg, uint64_t nbytes, int delimited, uint32_t n_train, uint32_t walk_ctas,
                                   uint32_t copy_ctas, uint8_t* out, uint64_t out_cap, uint32_t* rec_line,
                                   uint32_t* line_rec, uint32_t* line_dst, uint64_t* hdr) {
    std::vector<uint32_t> off, len;
    if (!delimited) { off.push_back(0); len.push_back((uint32_t)nbytes); }
    uint64_t pos = 0;
    while (delimited && pos < nbytes) {
        uint64_t l = 0;
        int shift = 0;
        for (;;) {
            if (pos >= nbytes || shift > 63) return -1;
            const uint8_t b = msg[pos++];
            l |= (uint64_t)(b & 0x7F) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (l > nbytes - pos) return -1;
        off.push_back((uint32_t)pos);
        len.push_back((uint32_t)l);
        pos += l;
    }
    const uint32_t n = (uint32_t)off.size();
    std::vector<uint8_t> buf(nbytes + 64, 0x0A);                     // hostile slack: '\n' bytes
    memcpy(buf.data(), msg, nbytes);
    const uint32_t tiles = (n + DML_THREADS - 1) / DML_THREADS;
    const uint32_t want = std::max<uint32_t>(1, std::min<uint32_t>(tiles, walk_ctas));
    const uint32_t per_cta = std::max<uint32_t>(1, (tiles + want - 1) / want) * DML_THREADS;
    const uint32_t n_chunks = (n + per_cta - 1) / per_cta;
    std::vector<uint32_t> text_off(n + 1), text_len(n + 1), line_src(n + 1);
    std::vector<unsigned long long> loc(n + 1), chunk(n_chunks + 1);
    DmLogsHeader lh;
    memset(&lh, 0, sizeof(lh));
    DmLogsArgs a;
    a.buf = buf.data(); a.rec_off = off.data(); a.rec_len = len.data(); a.n_records = n; a.n_train_records = n_train;
    a.per_cta = per_cta; a.n_chunks = n_chunks; a.text_off = text_off.data(); a.text_len = text_len.data();
    a.loc = loc.data(); a.chunk = chunk.data(); a.rec_line = rec_line; a.line_src = line_src.data(); a.line_dst = line_dst;
    a.line_rec = line_rec; a.out = out; a.out_cap = out_cap; a.lhdr = &lh;
    memset(out, 0xEE, out_cap);
    if (n) {
        emu_launch_grid(n_chunks, DML_THREADS, [&] { dm_k_logs_walk(a); });
        emu_launch_grid(1, DML_THREADS, [&] { dm_k_logs_scan(a); });
        emu_launch_grid(2, DML_THREADS, [&] { dm_k_logs_compact(a); });
        emu_launch_grid(copy_ctas, DML_THREADS, [&] { dm_k_logs_copy(a); });
    }
    hdr[0] = lh.total_bytes; hdr[1] = lh.n_lines; hdr[2] = lh.n_train; hdr[3] = lh.bound;
    return n;
}
