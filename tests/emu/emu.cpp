// emu.cpp -- runs the product's kernel sources (dm_kernels_*.cuh) on the CPU emulator.  TEST INFRASTRUCTURE ONLY:
// built by tests/emu_harness.py into tests/emu/_build/; never part of libdmdetect.so.
//
// Each emu_process_* / emu_* entry point enqueues the launches its libdmdetect counterpart enqueues, with the same
// host-side set-up (the arguments, the instantiation, the grid -- capped small here so that the kernels take their
// stride loops -- the framing and the anomaly merge all come from the kernel headers and dm_host.h).  Only the launch
// calls and the buffers differ: every scratch array and the bytes behind the message start out hostile.
#include "cuda_emu.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <type_traits>

#include "dm_kernels_index.cuh"
#include "dm_kernels_stream.cuh"
#include "dm_kernels_records.cuh"
#include "dm_kernels_format.cuh"
#include "dm_kernels_lanes.cuh"
#include "dm_kernels_logs.cuh"
#include "dm_kernels_alerts.cuh"
#include "dm_format_host.h"
#include "dm_host.h"

thread_local emu_dim3 threadIdx;
thread_local emu_dim3 blockIdx;
emu_dim3 blockDim, gridDim;
EmuBlock* g_emu_block = nullptr;
std::atomic<int> g_emu_or_flag[2];
std::vector<uint8_t> g_emu_dyn_smem;

// Runs the blocks of a grid ONE AFTER THE OTHER (block b sees blocks < b complete, which
// satisfies the look-back dependencies of the kernels under test).
void emu_launch_grid(unsigned blocks, unsigned threads, const std::function<void()>& body) {
    blockDim.x = threads;
    gridDim.x = blocks;
    for (unsigned b = 0; b < blocks; ++b) {
        EmuBlock blk;
        blk.warps = std::vector<EmuWarp>(threads / 32);
        g_emu_block = &blk;
        std::vector<std::thread> ts;
        ts.reserve(threads);
        for (unsigned t = 0; t < threads; ++t)
            ts.emplace_back([t, b, &body] {
                threadIdx.x = t;
                blockIdx.x = b;
                body();
            });
        for (auto& t : ts) t.join();
        g_emu_block = nullptr;
    }
}

void emu_launch(unsigned threads, const std::function<void()>& body) { emu_launch_grid(1, threads, body); }

// The emulated dm_handle: the known set, statistics, batch header and anomaly list, K_A's scratch, and the
// configuration the emu_set_* calls leave (as dm_set_monitors / dm_set_combos / dm_set_format / dm_set_alert_format).
struct EmuHandle {
    DmKeys keys;
    DmTable table;
    std::vector<unsigned long long> slots, novel;
    unsigned long long counts[2] = {0, 0};
    unsigned long long stats[DM_STATS_WORDS] = {0};
    DmBatchHeader hdr;
    std::vector<dm_anomaly_t> anoms;
    uint64_t max_lines = 0;
    std::vector<uint32_t> row_prefix;
    std::vector<unsigned long long> rows_tile_state;
    uint32_t rows_epoch = 0;
    DmMonitors mons{};                   // monitors and combinations
    DmFormat fmt{};
    bool fmt_set = false;
    std::string fmt_err;
    DmAlertFmt afmt{};
    bool afmt_set = false;
    struct EmuStream* xs = nullptr;      // stream variant (created on first use)
};

extern "C" EmuHandle* emu_create(uint32_t n_keys, const uint8_t* blob, const uint32_t* lens, uint32_t table_log2,
                                 uint64_t max_tiles, uint64_t max_lines) {
    EmuHandle* h = new EmuHandle();
    memset(&h->keys, 0, sizeof(DmKeys));
    h->keys.n = n_keys;
    uint64_t off = 0;
    for (uint32_t k = 0; k < n_keys; ++k) {
        h->keys.len[k] = lens[k];
        memcpy(h->keys.bytes[k], blob + off, lens[k]);
        h->keys.salt[k] = dm_field_salt(k);
        off += lens[k];
    }
    dm_keys_finalize_host(&h->keys);
    const uint64_t cap = 1ull << table_log2;
    h->slots.assign(cap, 0);
    h->novel.assign(cap / 2, 0);
    h->table.slots = h->slots.data();
    h->table.mask = (uint32_t)(cap - 1);
    h->table.limit = (uint32_t)(cap / 2);
    h->table.count = &h->counts[0];
    h->table.novel = h->novel.data();
    h->table.novel_count = &h->counts[1];
    h->table.novel_cap = (uint32_t)(cap / 2);
    (void)max_tiles;
    h->anoms.resize(1 << 16);
    h->max_lines = max_lines;
    memset(&h->hdr, 0, sizeof(h->hdr));
    return h;
}

void emu_stream_free(struct EmuStream*);
extern "C" void emu_destroy(EmuHandle* h) { emu_stream_free(h->xs); delete h; }

// as dm_set_monitors (which also clears the combinations)
extern "C" void emu_set_monitors(EmuHandle* h, const DmMonitor* mons, uint32_t n_mons) {
    memset(&h->mons, 0, sizeof(h->mons));
    h->mons.n = n_mons;
    for (uint32_t i = 0; i < n_mons; ++i) h->mons.m[i] = mons[i];
}

// as dm_set_combos (0 combinations = off)
extern "C" void emu_set_combos(EmuHandle* h, uint32_t n_combos, const uint32_t* member_off, const uint32_t* members,
                               uint32_t member_only) {
    DmMonitors& m = h->mons;
    m.n_combos = n_combos;
    m.member_only = member_only;
    memset(m.combo_off, 0, sizeof(m.combo_off));
    memset(m.combo_members, 0, sizeof(m.combo_members));
    for (uint32_t c = 0; n_combos && c <= n_combos; ++c) m.combo_off[c] = member_off[c];
    for (uint32_t j = 0; n_combos && j < member_off[n_combos]; ++j) m.combo_members[j] = (uint8_t)members[j];
}

// as dm_set_format_ex, binding the monitors of emu_set_monitors; nullptr or the reason it refuses
extern "C" const char* emu_set_format(EmuHandle* h, const char* log_format, const char* content_name, uint32_t n_templates,
                                      const char* const* templates, uint32_t norm_flags) {
    h->fmt_err.clear();
    h->fmt_set = dm_format_build(log_format, content_name, n_templates, templates, norm_flags, h->mons, &h->fmt, &h->fmt_err);
    return h->fmt_set ? nullptr : h->fmt_err.c_str();
}

// The message in a 64-byte aligned buffer, followed by 64 hostile bytes (slack, repeated).
static uint8_t* emu_message(const uint8_t* msg, uint64_t nbytes, const std::vector<uint8_t>& slack) {
    uint8_t* buf = (uint8_t*)aligned_alloc(64, ((nbytes + 64 + 63) / 64) * 64 + 64);
    memcpy(buf, msg, nbytes);
    for (uint32_t i = 0; i < 64; ++i) buf[nbytes + i] = slack[i % slack.size()];
    return buf;
}
static const std::vector<uint8_t> EMU_KV_SLACK = {'=', '\n'};

// ---------------------------------------------------------------------------------------------- stream kernel
// As dmx_launch: [row counts, boundary, TRAIN launch,] DETECT launch.  The grid is capped at `g_emu_stream_ctas` CTAs
// run one after the other (the last one runs the epilogue).
static uint32_t g_emu_stream_ctas = 3;
extern "C" void emu_stream_ctas(uint32_t n) { g_emu_stream_ctas = n ? n : 1; }
struct EmuStream {
    DmxKeyTab tab;
    DmxShared sh;
    std::vector<unsigned short> row_cnt[DMX_NPAR], bound_cnt;
    std::vector<unsigned int> cta_cnt[DMX_NPAR];
    std::vector<dm_anomaly_t> alerts[DMX_NPAR];
    unsigned int alert_count[DMX_NPAR] = {};
    unsigned long long bound = 0, seq = 0, hint = 0;
    bool ready = false;
};
static unsigned long long g_emu_last_hint = 0;
void emu_stream_free(EmuStream* x) { delete x; }
static int emu_stream_run(EmuHandle* h, bool chained, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                          float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    if (!h->xs) {
        h->xs = new EmuStream();
        if (!dmx_keytab_build(h->keys, &h->xs->tab)) return -7;
        memset(&h->xs->sh, 0, sizeof(h->xs->sh));
    }
    EmuStream& g_xs = *h->xs;
    // as dm_process_lines: the header is the previous call's until this call's epilogue rewrites it (its take-out of
    // the previous call's alerts reads it), except for an empty message; errors are read as dm_sync reads them
    *n_lines = 0; *n_anoms = 0; *err = 0;
    const uint32_t n_rows = (uint32_t)((nbytes + DMX_ROW - 1) / DMX_ROW);
    if (n_rows == 0) {
        memset(&h->hdr, 0, sizeof(h->hdr));
        *err = g_xs.sh.error;
        g_xs.sh.error = 0;
        return 0;
    }
    uint8_t* buf = emu_message(msg, nbytes, EMU_KV_SLACK);
    for (unsigned b = 0; b < DMX_NPAR; ++b) {
        if (g_xs.row_cnt[b].size() < n_rows + 1) g_xs.row_cnt[b].assign(n_rows + 1, 0xBEEF);
        if (g_xs.alerts[b].size() < h->anoms.size()) g_xs.alerts[b].resize(h->anoms.size());
        g_xs.cta_cnt[b].assign(g_emu_stream_ctas + 1, 0xDEADBEEFu);
    }
    g_xs.bound_cnt.assign(n_rows + 1, 0xBEEF);
    g_emu_dyn_smem.assign(DMX_RING_SMEM + sizeof(DmxKeyTab), 0xEE);
    DmxArgs a;
    a.buf = buf; a.nbytes = nbytes; a.n_rows = n_rows; a.keys = &g_xs.tab; a.table = h->table;
    a.flags = flags; a.scores = scores; a.out_cap = cap; a.anomalies = h->anoms.data(); a.anomaly_cap = (uint32_t)h->anoms.size();
    a.hdr = &h->hdr; a.stats = h->stats; a.n_train_lines = n_train; a.max_lines = h->max_lines;
    a.sh = &g_xs.sh; a.alert_cap = (uint32_t)h->anoms.size(); a.bound_ptr = nullptr; a.keep_error = 0; a.timeline = nullptr; a.ring_smem = DMX_RING_SMEM;
    a.hint = &g_xs.hint;
    a.error_acc = &g_xs.sh.error;
    a.keytab_bytes = (uint32_t)((DMX_KEYTAB_HOT(g_xs.tab.l1_slots) + 15) & ~(size_t)15);
    const unsigned grid = dmx_geometry(a, g_emu_stream_ctas);
    auto bind = [&]() {
        a.seq = ++g_xs.seq;
        const int p = (int)(a.seq % DMX_NPAR);
        a.row_cnt = g_xs.row_cnt[p].data(); a.cta_cnt = g_xs.cta_cnt[p].data(); a.alerts = g_xs.alerts[p].data(); a.alert_count = &g_xs.alert_count[p];
    };
    if (n_train > 0) {
        const uint32_t b_rows = (uint32_t)((nbytes + DMB_ROW - 1) / DMB_ROW);
        g_xs.bound_cnt.assign(b_rows + 1, 0xBEEF);
        emu_launch_grid(2, 256, [&] { dm_k_rowcount(buf, nbytes, b_rows, g_xs.bound_cnt.data()); });
        emu_launch(256, [&] { dm_k_bound(buf, nbytes, b_rows, g_xs.bound_cnt.data(), n_train, &g_xs.bound, &h->hdr); });
        a.bound_ptr = &g_xs.bound; a.keep_error = 1;
        bind();
        if (chained) emu_launch_grid(grid, DMX_THREADS, [&] { dm_k_stream<true, true>(a); });
        else emu_launch_grid(grid, DMX_THREADS, [&] { dm_k_stream<true, false>(a); });
    }
    bind();
    if (chained) emu_launch_grid(grid, DMX_THREADS, [&] { dm_k_stream<false, true>(a); });
    else emu_launch_grid(grid, DMX_THREADS, [&] { dm_k_stream<false, false>(a); });
    g_emu_last_hint = g_xs.hint;
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error | g_xs.sh.error;
    g_xs.sh.error = 0;
    return 0;
}

// the two instantiations of the stream kernel: candidates re-checked one by one / batch-wise (dmx_verify_chain)
extern "C" int emu_process_stream(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                  float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    return emu_stream_run(h, false, msg, nbytes, n_train, flags, scores, cap, n_lines, n_anoms, err);
}
extern "C" int emu_process_stream_chain(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                        float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    return emu_stream_run(h, true, msg, nbytes, n_train, flags, scores, cap, n_lines, n_anoms, err);
}
// what the last detect launch told the host: (batches with a candidate << 32) | rows
extern "C" unsigned long long emu_stream_hint(void) { return g_emu_last_hint; }

extern "C" void emu_chain_stats(unsigned long long* out, int reset) {
    for (int i = 0; i < 8; ++i) { out[i] = g_emu_chain_stats[i]; if (reset) g_emu_chain_stats[i] = 0; }
}

// ---------------------------------------------------------------------------------------------- thread per record
// K_A (the record index and the batch header), then the train launch (n_train > 0) and the detect launch of a
// thread-per-record kernel, as dm_lanes_launch and the format branch of dm_process_lines enqueue them.  launch(train,
// args) runs one of the two.
template <typename Launch>
static void emu_per_record(EmuHandle* h, const uint8_t* buf, uint64_t nbytes, uint64_t n_train, uint8_t* flags, float* scores,
                           uint64_t cap, const void* combos, Launch launch) {
    std::vector<uint32_t> ls(h->max_lines + 2, 0xDEADBEEFu);
    DmRowsArgs ra = dm_rows_args(buf, nbytes, nullptr, nullptr, &h->rows_epoch, ls.data(), flags, scores, cap, &h->hdr,
                                 h->stats, n_train, h->max_lines);
    h->row_prefix.assign(ra.n_rows + 1, 0xDEADBEEFu);
    if (h->rows_tile_state.size() < ra.n_tiles + 1) h->rows_tile_state.resize(ra.n_tiles + 1, 0);
    ra.row_prefix = h->row_prefix.data();
    ra.tile_state = h->rows_tile_state.data();
    emu_launch_grid(ra.n_tiles, DMR_A_THREADS, [&] { dm_k_rowindex(ra); });
    DmDetectArgs a = dm_detect_args(buf, nbytes, ls.data(), &h->hdr, &h->keys, h->table, flags, scores, cap, h->anoms.data(),
                                    (uint32_t)h->anoms.size(), h->stats, combos);
    if (n_train > 0) {
        a.line_lo = 0; a.line_hi = n_train;
        launch(true, a);
    }
    a.line_lo = n_train; a.line_hi = ~0ull;
    launch(false, a);
}

// key=value records, one thread each (dm_kernels_lanes.cuh), on at most 5 CTAs
extern "C" int emu_process_lanes(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                 float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    *n_lines = 0; *n_anoms = 0; *err = 0;
    if (nbytes == 0) { memset(&h->hdr, 0, sizeof(h->hdr)); return 0; }      // as dm_process_lines: no launch at all
    uint8_t* buf = emu_message(msg, nbytes, EMU_KV_SLACK);
    const bool combo = h->mons.n_combos > 0;
    const unsigned grid = dm_detect_grid(nbytes, h->max_lines, DM_LANES_THREADS, 5);
    g_emu_dyn_smem.assign((size_t)DM_MAX_KEYS * DM_LANES_THREADS * sizeof(unsigned long long), 0);
    emu_per_record(h, buf, nbytes, n_train, flags, scores, cap, combo ? &h->mons : nullptr, [&](bool train, const DmDetectArgs& a) {
        const DmLanesKernel k = dm_lanes_kernel(train, combo);
        emu_launch_grid(grid, DM_LANES_THREADS, [&] { k(a); });
    });
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error;
    return 0;
}

// log_format / template mode (dm_kernels_format.cuh), with the combinations of emu_set_combos if any, on at most 3 CTAs
// (messages of more than 192 records take the kernel's stride loop)
extern "C" int emu_process_format(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                  float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    if (!h->fmt_set) return -6;
    *n_lines = 0; *n_anoms = 0; *err = 0;
    if (nbytes == 0) { memset(&h->hdr, 0, sizeof(h->hdr)); return 0; }      // as dm_process_lines: no launch at all
    const DmFormat& f = h->fmt;
    // hostile slack: the bytes of the configured literals, each followed by '\n', over and over (the kernel reads up to
    // 12 bytes past a record; none of it may count)
    std::vector<uint8_t> slack;
    for (uint32_t i = 0; i < f.chain_first[f.n_chains]; ++i) {
        for (uint32_t j = 0; j < f.lit_len[i]; ++j) slack.push_back((uint8_t)(f.pool[f.lit_off[i] + j / 4] >> (8 * (j % 4))));
        slack.push_back('\n');
    }
    uint8_t* buf = emu_message(msg, nbytes, slack);
    // R-norm scratch: hostile content (the kernel may only read back what it wrote itself)
    uint8_t* nbuf = (uint8_t*)aligned_alloc(64, ((nbytes + 256 + 63) / 64) * 64);
    memset(nbuf, 0xA5, nbytes + 256);
    const bool norm = dm_format_norm(f), combo = h->mons.n_combos > 0;
    const unsigned grid = dm_detect_grid(nbytes, h->max_lines, DM_FMTL_THREADS, 3);
    g_emu_dyn_smem.assign((size_t)2 * f.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
    emu_per_record(h, buf, nbytes, n_train, flags, scores, cap, combo ? &h->mons : nullptr, [&](bool train, const DmDetectArgs& a) {
        const DmFormatLanesKernel k = dm_format_lanes_kernel(train, norm, combo);
        emu_launch_grid(grid, DM_FMTL_THREADS, [&] { k(a, &f, nbuf); });
    });
    free(nbuf);
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error;
    return 0;
}

// ---------------------------------------------------------------------------------------------- records
// The framing split of dm_process_records / dm_process_logs: the record count (offsets / lengths of the first cap
// records in off / len), or -DM_FRAME_* with *at = the byte where the error was found.
extern "C" int64_t emu_frame_split(const uint8_t* buf, uint64_t nbytes, uint32_t* off, uint32_t* len, uint64_t cap, uint64_t* at) {
    const DmFrames fr = dm_frame_split(buf, nbytes);
    *at = fr.at;
    if (fr.error) return -fr.error;
    for (uint64_t i = 0; i < fr.off.size() && i < cap; ++i) { off[i] = fr.off[i]; len[i] = fr.len[i]; }
    return (int64_t)fr.off.size();
}

// ParserSchema records, as dm_process_records: the host framing, then the train / bound / detect launches of
// dm_k_records with the monitors and combinations of emu_set_monitors / emu_set_combos.  -1: a framing error.
extern "C" int emu_process_records(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint32_t n_train, uint8_t* flags,
                                   float* scores, uint32_t* masks, uint64_t cap, uint64_t* n_records, uint64_t* n_anoms) {
    const DmFrames fr = dm_frame_split(msg, nbytes);
    if (fr.error) return -1;
    const uint32_t n = (uint32_t)fr.off.size();
    if (n > cap) return -4;
    memset(&h->hdr, 0, sizeof(h->hdr));
    DmRecordsArgs a;
    a.buf = msg; a.rec_off = fr.off.data(); a.rec_len = fr.len.data(); a.n_records = n; a.n_train_records = n_train;
    a.mons = &h->mons; a.table = h->table; a.flags = flags; a.scores = scores; a.masks = masks; a.hdr = &h->hdr; a.stats = h->stats;
    uint32_t bound[2] = {0, 0};
    if (n) {
        if (n_train > 0) {
            emu_launch(128, [&] { dm_k_records(a, 2); });
            emu_launch(256, [&] { dm_k_records_bound(flags, n, n_train, bound); });
            emu_launch(128, [&] { dm_k_records(a, 0, bound); });
        }
        if (n_train < n) emu_launch(128, [&] { dm_k_records(a, 1, n_train > 0 ? bound : nullptr); });
    }
    dm_stats_add_records(h->stats, n, bound[1], n - (n_train > 0 ? bound[0] : 0), nbytes);
    *n_records = n;
    *n_anoms = h->hdr.n_anomalies;
    return 0;
}

// ---------------------------------------------------------------------------------------------- LogSchema unwrap
// Frames the message as dm_process_logs does, then runs the four unwrap kernels (dm_kernels_logs.cuh) with the walk
// grid capped at `walk_ctas` CTAs (so that a CTA walks several tiles of records) and the copy on `copy_ctas` CTAs (so
// that its threads take the grid-stride loop).  The message is followed by hostile bytes, the output buffer is
// pre-filled with 0xEE.  Outputs: out (the compacted texts and the slack), rec_line / line_rec / line_dst, hdr =
// {total_bytes, n_lines, n_train, bound}.  Returns the record count, or -1 for a framing error.
extern "C" int64_t emu_logs_unwrap(const uint8_t* msg, uint64_t nbytes, int delimited, uint32_t n_train, uint32_t walk_ctas,
                                   uint32_t copy_ctas, uint8_t* out, uint64_t out_cap, uint32_t* rec_line,
                                   uint32_t* line_rec, uint32_t* line_dst, uint64_t* hdr) {
    DmFrames fr;
    if (delimited) {
        fr = dm_frame_split(msg, nbytes);
        if (fr.error) return -1;
    } else {
        fr.off.push_back(0);
        fr.len.push_back((uint32_t)nbytes);
    }
    const uint32_t n = (uint32_t)fr.off.size();
    std::vector<uint8_t> buf(nbytes + 64, 0x0A);                     // hostile slack: '\n' bytes
    memcpy(buf.data(), msg, nbytes);
    uint32_t per_cta;
    const uint32_t n_chunks = dm_logs_plan(n, walk_ctas, &per_cta);
    std::vector<uint32_t> text_off(n + 1), text_len(n + 1), line_src(n + 1);
    std::vector<unsigned long long> loc(n + 1), chunk(n_chunks + 1);
    DmLogsHeader lh;
    memset(&lh, 0, sizeof(lh));
    DmLogsArgs a;
    a.buf = buf.data(); a.rec_off = fr.off.data(); a.rec_len = fr.len.data(); a.n_records = n; a.n_train_records = n_train;
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

// ---------------------------------------------------------------------------------------------- DetectorSchema alerts
// as dm_set_alert_format (the monitors' keys are those of emu_create); nullptr or the reason it refuses
extern "C" const char* emu_set_alert_format(EmuHandle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* lens,
                                            const uint32_t* bits_off, const uint32_t* bits, uint32_t n_combos,
                                            const uint32_t* combo_off, const uint32_t* members, uint32_t time_cap) {
    const char* why = dm_alert_fmt_build(h->keys, n_strings, strings, lens, bits_off, bits, n_combos, combo_off, members,
                                         time_cap, &h->afmt);
    h->afmt_set = why == nullptr;
    return why;
}

// As dm_encode_alerts on the last batch: msg / scores are that batch's message and scores (the emulated detect
// functions do not keep them); fmt: the batch was detected in log_format mode (emu_set_format's format).  The
// grid-stride kernels run on 2 CTAs, so that batches of more than 512 (log_format: 128) anomaly entries take their
// stride loops; every scratch array, the R-norm scratch included, starts out hostile.  Returns 0, or -6 without an alert
// format.
extern "C" int emu_encode_alerts(EmuHandle* h, int fmt, const uint8_t* msg, uint64_t nbytes, const float* scores,
                                 uint64_t first_log_id, int64_t first_alert_id, int64_t now, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    if (!h->afmt_set) return -6;
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
    a.fmt = &h->afmt; a.buf = buf.data(); a.nbytes = nbytes; a.scores = scores; a.anoms = h->anoms.data();
    a.n_entries = entries; a.n_lines = n_lines; a.rank = rank.data(); a.rec_line = rec_line.data(); a.rec_mask = rec_mask.data();
    a.rec_off = rec_off.data(); a.size = size.data(); a.ahdr = &ah; a.first_log_id = first_log_id;
    a.first_alert_id = first_alert_id; a.now = now; a.out = dout.data(); a.out_cap = out_cap;
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

// ---------------------------------------------------------------------------------------------- read-back
// as dm_get_anomalies: the batch's entries merged per record, at most cap of them; their count
extern "C" uint32_t emu_get_anomalies(EmuHandle* h, dm_anomaly_t* out, uint32_t cap) {
    const uint32_t n = std::min<uint32_t>(h->hdr.anomaly_list_count, (uint32_t)h->anoms.size());
    std::vector<dm_anomaly_t> v(h->anoms.begin(), h->anoms.begin() + n);
    const uint32_t m = std::min(dm_anomalies_merge(v.data(), n), cap);
    std::copy(v.begin(), v.begin() + m, out);
    return m;
}

extern "C" void emu_get_stats(EmuHandle* h, unsigned long long* out) {
    for (int i = 0; i < DM_STATS_WORDS; ++i) out[i] = h->stats[i];
    out[6] = h->counts[0];
}

extern "C" uint64_t emu_export_known(EmuHandle* h, unsigned long long* out, uint64_t cap) {
    uint64_t n = std::min<uint64_t>(h->counts[1], h->novel.size());
    std::vector<unsigned long long> v(h->novel.begin(), h->novel.begin() + n);
    std::sort(v.begin(), v.end());
    for (uint64_t i = 0; i < n && i < cap; ++i) out[i] = v[i];
    return n;
}
