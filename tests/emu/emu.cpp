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
#include "dm_kernels_parse.cuh"
#include "dm_kernels_window.cuh"
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

// The emulated dm_handle: the known set, statistics, batch header and anomaly list, K_A's scratch, the configuration
// the emu_set_* calls leave (as dm_set_monitors / dm_set_combos / dm_set_format / dm_set_alert_format /
// dm_set_parser_format), and what the last batch leaves for the encoder.
struct EmuHandle {
    DmKeys keys;
    DmTable table;
    std::vector<unsigned long long> slots, novel;
    unsigned long long counts[2] = {0, 0};
    unsigned long long stats[DM_STATS_WORDS] = {0};
    unsigned long long stats_exported[DM_STATS_WORDS] = {0};   // the window exchange (dm_handle::d_stats_exported,
    unsigned long long stats_global[DM_STATS_WORDS] = {0};     //   d_stats_global, novel_exported, novel_pending)
    uint64_t novel_exported = 0, novel_pending = 0;
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
    DmFormat efmt{};                     // the encoder's format (dm_alert_efmt_build), once fmt and afmt are set
    DmParseFmt pf{};                     // the parser's format and the matcher's format it runs (dm_parse_efmt_build)
    DmFormat pfmt{};
    bool parse_set = false;              // cleared by emu_set_format, as by dm_set_format
    struct EmuStream* xs = nullptr;      // stream variant (created on first use)
    // the last batch, as dm_encode_alerts reads it: its source (DMA_*), the message the line path read (emu_message),
    // its scores, the ParserSchema records; a LogSchema or ParserSchema message with hostile slack (d_in), the record
    // frames, flags, scores and masks of dm_process_records (d_vals, d_flags, d_scores, d_masks)
    uint32_t last_src = DMA_SRC_NONE;
    uint8_t* msg = nullptr;
    uint64_t msg_bytes = 0;
    const float* last_scores = nullptr;
    uint32_t last_n_records = 0;
    std::vector<uint8_t> in, flags;
    std::vector<float> scores;
    std::vector<uint32_t> vals, masks;
    // the unwrap of the last LogSchema message: its arrays (one block, dm_logs_carve), header and compacted texts
    std::vector<uint8_t> logs, logs_text;
    uint64_t logs_cap = 0;
    uint32_t logs_chunks = 0;
    DmLogsHeader lhdr;
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
extern "C" void emu_destroy(EmuHandle* h) {
    emu_stream_free(h->xs);
    free(h->msg);
    delete h;
}

// the anomaly list's capacity (dm_handle::anomaly_cap; 65536 from emu_create)
extern "C" void emu_set_anomaly_cap(EmuHandle* h, uint32_t cap) { h->anoms.assign(cap ? cap : 1, dm_anomaly_t{}); }

// as dm_alert_efmt_upload: the encoder's copy of the log_format, once both formats are set
static void emu_efmt_build(EmuHandle* h) {
    if (h->fmt_set && h->afmt_set) dm_alert_efmt_build(h->fmt, h->afmt.time_cap, &h->efmt);
}

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
    if (!h->fmt_set) return h->fmt_err.c_str();
    h->parse_set = false;
    emu_efmt_build(h);
    return nullptr;
}

// The message in a 64-byte aligned buffer, followed by 64 hostile bytes (slack, repeated); the handle keeps it as the
// batch the line path read (dm_handle::last_buf / last_nbytes).
static uint8_t* emu_message(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, const std::vector<uint8_t>& slack) {
    free(h->msg);
    uint8_t* buf = (uint8_t*)aligned_alloc(64, ((nbytes + 64 + 63) / 64) * 64 + 64);
    if (nbytes) memcpy(buf, msg, nbytes);
    for (uint32_t i = 0; i < 64; ++i) buf[nbytes + i] = slack[i % slack.size()];
    h->msg = buf;
    h->msg_bytes = nbytes;
    return buf;
}

// What dm_process_lines leaves for dm_encode_alerts besides the message: the batch's scores (copied: the caller's
// arrays need not outlive the call) and its source.
static void emu_lines_kept(EmuHandle* h, const float* scores, uint64_t cap) {
    h->scores.assign(scores, scores + std::min<uint64_t>(h->hdr.n_lines, cap));
    h->last_scores = h->scores.data();
    h->last_src = DMA_LINES;
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
        emu_message(h, msg, 0, EMU_KV_SLACK);
        emu_lines_kept(h, scores, 0);
        *err = g_xs.sh.error;
        g_xs.sh.error = 0;
        return 0;
    }
    uint8_t* buf = emu_message(h, msg, nbytes, EMU_KV_SLACK);
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
    emu_lines_kept(h, scores, cap);
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
    uint8_t* buf = emu_message(h, msg, nbytes, EMU_KV_SLACK);
    if (nbytes == 0) {                                                        // as dm_process_lines: no launch at all
        memset(&h->hdr, 0, sizeof(h->hdr));
        emu_lines_kept(h, scores, 0);
        return 0;
    }
    const bool combo = h->mons.n_combos > 0;
    const unsigned grid = dm_detect_grid(nbytes, h->max_lines, DM_LANES_THREADS, 5);
    g_emu_dyn_smem.assign((size_t)DM_MAX_KEYS * DM_LANES_THREADS * sizeof(unsigned long long), 0);
    emu_per_record(h, buf, nbytes, n_train, flags, scores, cap, combo ? &h->mons : nullptr, [&](bool train, const DmDetectArgs& a) {
        const DmLanesKernel k = dm_lanes_kernel(train, combo);
        emu_launch_grid(grid, DM_LANES_THREADS, [&] { k(a); });
    });
    emu_lines_kept(h, scores, cap);
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
    if (nbytes == 0) {                                                        // as dm_process_lines: no launch at all
        memset(&h->hdr, 0, sizeof(h->hdr));
        emu_message(h, msg, 0, EMU_KV_SLACK);
        emu_lines_kept(h, scores, 0);
        return 0;
    }
    const DmFormat& f = h->fmt;
    // hostile slack: the bytes of the configured literals, each followed by '\n', over and over (the kernel reads up to
    // 12 bytes past a record; none of it may count)
    std::vector<uint8_t> slack;
    for (uint32_t i = 0; i < f.chain_first[f.n_chains]; ++i) {
        for (uint32_t j = 0; j < f.lit_len[i]; ++j) slack.push_back((uint8_t)(f.pool[f.lit_off[i] + j / 4] >> (8 * (j % 4))));
        slack.push_back('\n');
    }
    uint8_t* buf = emu_message(h, msg, nbytes, slack);
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
    emu_lines_kept(h, scores, cap);
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
// dm_k_records with the monitors and combinations of emu_set_monitors / emu_set_combos, on the handle's copy of the
// message and arrays (hostile to start with), the outputs then copied to flags / scores / masks.  -1: a framing error.
extern "C" int emu_process_records(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint32_t n_train, uint8_t* flags,
                                   float* scores, uint32_t* masks, uint64_t cap, uint64_t* n_records, uint64_t* n_anoms) {
    const DmFrames fr = dm_frame_split(msg, nbytes);
    if (fr.error) return -1;
    const uint32_t n = (uint32_t)fr.off.size();
    if (n > cap) return -4;
    h->last_src = DMA_SRC_NONE;
    memset(&h->hdr, 0, sizeof(h->hdr));
    h->in.assign(nbytes + 64, 0x0A);                                // hostile slack: '\n' bytes
    if (nbytes) memcpy(h->in.data(), msg, nbytes);
    h->vals = fr.off;                                                // offsets, then lengths (as d_vals)
    h->vals.insert(h->vals.end(), fr.len.begin(), fr.len.end());
    h->flags.assign(n + 1, 7);
    h->scores.assign(n + 1, -1.0f);
    h->masks.assign(n + 1, 0xDEADBEEFu);
    DmRecordsArgs a;
    a.buf = h->in.data(); a.rec_off = h->vals.data(); a.rec_len = h->vals.data() + n; a.n_records = n; a.n_train_records = n_train;
    a.mons = &h->mons; a.table = h->table; a.flags = h->flags.data(); a.scores = h->scores.data(); a.masks = h->masks.data();
    a.hdr = &h->hdr; a.stats = h->stats;
    uint32_t bound[2] = {0, 0};
    if (n) {
        if (n_train > 0) {
            emu_launch(128, [&] { dm_k_records(a, 2); });
            emu_launch(256, [&] { dm_k_records_bound(h->flags.data(), n, n_train, bound); });
            emu_launch(128, [&] { dm_k_records(a, 0, bound); });
        }
        if (n_train < n) emu_launch(128, [&] { dm_k_records(a, 1, n_train > 0 ? bound : nullptr); });
    }
    dm_stats_add_records(h->stats, n, bound[1], n - (n_train > 0 ? bound[0] : 0), nbytes);
    memcpy(flags, h->flags.data(), n);
    memcpy(scores, h->scores.data(), (uint64_t)n * 4);
    memcpy(masks, h->masks.data(), (uint64_t)n * 4);
    *n_records = n;
    *n_anoms = h->hdr.n_anomalies;
    h->last_src = DMA_RECORDS;
    h->last_n_records = n;
    h->last_scores = h->scores.data();
    return 0;
}

// ---------------------------------------------------------------------------------------------- LogSchema unwrap
// As dm_logs_unwrap, for the records fr of the message: the handle keeps the message with hostile slack ('\n' bytes)
// and the unwrap's arrays, carved from one block that is filled with hostile bytes before each call.  The walk runs on
// at most walk_ctas CTAs, the compact on at most 2 and (when out is set) the copy on at most copy_ctas, so that a CTA
// walks several tiles of records and the others take their grid-stride loops.
static void emu_unwrap(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, const DmFrames& fr, uint32_t n_train,
                       uint32_t walk_ctas, uint32_t copy_ctas, uint8_t* out, uint64_t out_cap, DmLogsArgs* a,
                       float** rscores, uint8_t** rflags) {
    const uint32_t n = (uint32_t)fr.off.size();
    h->in.assign(nbytes + 64, 0x0A);
    if (nbytes) memcpy(h->in.data(), msg, nbytes);
    h->logs_cap = n;
    h->logs_chunks = walk_ctas;
    h->logs.assign(dm_logs_scratch_bytes(h->logs_cap, h->logs_chunks), 0xEE);
    memset(&h->lhdr, 0xEE, sizeof(h->lhdr));
    *a = dm_logs_carve(h->logs.data(), h->logs_cap, h->logs_chunks, &h->lhdr, rscores, rflags);
    dm_logs_call(a, h->in.data(), n, n_train, walk_ctas, out, out_cap);
    std::copy(fr.off.begin(), fr.off.end(), (uint32_t*)a->rec_off);
    std::copy(fr.len.begin(), fr.len.end(), (uint32_t*)a->rec_len);
    if (n) {
        emu_launch_grid(a->n_chunks, DML_THREADS, [&] { dm_k_logs_walk(*a); });
        emu_launch_grid(1, DML_THREADS, [&] { dm_k_logs_scan(*a); });
        emu_launch_grid(dm_grid(n, DML_THREADS, 2), DML_THREADS, [&] { dm_k_logs_compact(*a); });
        if (out) emu_launch_grid(dm_logs_copy_grid(nbytes, copy_ctas), DML_THREADS, [&] { dm_k_logs_copy(*a); });
    } else {
        memset(&h->lhdr, 0, sizeof(h->lhdr));                         // as dm_logs_unwrap's cudaMemsetAsync of d_lhdr
    }
}

// The unwrap kernels alone: frames the message as dm_process_logs does and unwraps it (the walk on at most `walk_ctas`
// CTAs, the copy on at most `copy_ctas`) into out, pre-filled with 0xEE.  Outputs: out (the compacted texts and the
// slack), rec_line / line_rec / line_dst, hdr = {total_bytes, n_lines, n_train, bound}.  Returns the record count, or -1
// for a framing error.
extern "C" int64_t emu_logs_unwrap(const uint8_t* msg, uint64_t nbytes, int delimited, uint32_t n_train, uint32_t walk_ctas,
                                   uint32_t copy_ctas, uint8_t* out, uint64_t out_cap, uint32_t* rec_line,
                                   uint32_t* line_rec, uint32_t* line_dst, uint64_t* hdr) {
    const DmFrames fr = dm_frame_records(msg, nbytes, delimited != 0);
    if (fr.error) return -1;
    EmuHandle* h = new EmuHandle();
    memset(out, 0xEE, out_cap);
    DmLogsArgs a;
    float* rscores;
    uint8_t* rflags;
    emu_unwrap(h, msg, nbytes, fr, n_train, walk_ctas, copy_ctas, out, out_cap, &a, &rscores, &rflags);
    const DmLogsHeader lh = h->lhdr;
    std::copy(a.rec_line, a.rec_line + a.n_records, rec_line);
    std::copy(a.line_rec, a.line_rec + lh.n_lines, line_rec);
    if (a.n_records) std::copy(a.line_dst, a.line_dst + lh.n_lines + 1, line_dst);
    hdr[0] = lh.total_bytes; hdr[1] = lh.n_lines; hdr[2] = lh.n_train; hdr[3] = lh.bound;
    emu_destroy(h);
    return a.n_records;
}

// As dm_process_logs: the framing, the unwrap (walk and copy on at most 2 CTAs), the line path of `variant` (0 stream,
// 1 stream with the chained re-check, 2 lanes, 3 log_format) on the compacted texts, then dm_k_logs_scatter on at most 2
// CTAs.  flags / scores: per record (cap entries).  Returns 0, -1 for a framing error, -4 when the records exceed cap,
// or the line path's error.
extern "C" int emu_process_logs(EmuHandle* h, int variant, const uint8_t* msg, uint64_t nbytes, int delimited, uint32_t n_train,
                                uint8_t* flags, float* scores, uint64_t cap, uint64_t* n_records, uint64_t* n_malformed,
                                uint64_t* n_anoms) {
    const DmFrames fr = dm_frame_records(msg, nbytes, delimited != 0);
    if (fr.error) return -1;
    const uint32_t n = (uint32_t)fr.off.size();
    if (n > cap) return -4;
    h->logs_text.assign(dm_logs_text_bytes(nbytes), 0xEE);
    DmLogsArgs a;
    float* rscores;
    uint8_t* rflags;
    emu_unwrap(h, msg, nbytes, fr, n_train, 2, 2, h->logs_text.data(), h->logs_text.size(), &a, &rscores, &rflags);
    const DmLogsHeader lh = h->lhdr;
    std::vector<uint8_t> lflags(lh.n_lines + 2, 7);
    std::vector<float> lscores(lh.n_lines + 2, -1.0f);
    if (lh.n_lines) {
        uint64_t nl = 0, na = 0;
        uint32_t err = 0;
        uint8_t* text = h->logs_text.data();
        int rc;
        if (variant <= 1) rc = emu_stream_run(h, variant == 1, text, lh.total_bytes, lh.n_train, lflags.data(), lscores.data(),
                                             lh.n_lines + 2, &nl, &na, &err);
        else if (variant == 2) rc = emu_process_lanes(h, text, lh.total_bytes, lh.n_train, lflags.data(), lscores.data(),
                                                      lh.n_lines + 2, &nl, &na, &err);
        else rc = emu_process_format(h, text, lh.total_bytes, lh.n_train, lflags.data(), lscores.data(), lh.n_lines + 2,
                                     &nl, &na, &err);
        h->last_src = DMA_SRC_NONE;                                      // (its anomaly list is rewritten to records below)
        if (rc != 0) return rc;
        if (err || nl != lh.n_lines) return -5;
    } else {
        memset(&h->hdr, 0, sizeof(h->hdr));
        h->last_src = DMA_SRC_NONE;
    }
    emu_launch_grid(dm_logs_scatter_grid(n, (uint32_t)h->anoms.size(), 2), DML_THREADS, [&] {
        dm_k_logs_scatter(a, lflags.data(), lscores.data(), rflags, rscores, h->anoms.data(), (uint32_t)h->anoms.size(),
                          &h->hdr, h->stats, nbytes);
    });
    memcpy(flags, rflags, n);
    memcpy(scores, rscores, (uint64_t)n * 4);
    *n_records = n;
    *n_malformed = n - lh.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    h->last_src = DMA_LOGS;                                              // (the line path left the message: the texts)
    h->last_scores = rscores;
    return 0;
}

// ---------------------------------------------------------------------------------------------- DetectorSchema alerts
// as dm_set_alert_format (the monitors' keys are those of emu_create); nullptr or the reason it refuses
extern "C" const char* emu_set_alert_format(EmuHandle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* lens,
                                            const uint32_t* bits_off, const uint32_t* bits, uint32_t n_combos,
                                            const uint32_t* combo_off, const uint32_t* members, uint32_t time_cap) {
    const char* why = dm_alert_fmt_build(h->keys, n_strings, strings, lens, bits_off, bits, n_combos, combo_off, members,
                                         time_cap, &h->afmt);
    h->afmt_set = why == nullptr;
    emu_efmt_build(h);
    return why;
}

// exclusive scan of d[0, n) as dm_alert_scan launches it; the sum to *total
template <typename T>
static void emu_scan(T* d, uint64_t n, T* tile_sums, T* total) {
    const uint32_t nt = (uint32_t)std::max<uint64_t>(1, dm_alert_tiles(n));
    emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_tiles<T>(d, n, tile_sums); });
    emu_launch(DMA_THREADS, [&] { dm_k_alert_scan_top<T>(tile_sums, nt, total); });
    emu_launch_grid(nt, DMA_THREADS, [&] { dm_k_alert_scan_apply<T>(d, n, tile_sums); });
}

// As dm_encode_alerts on the last batch of emu_process_stream / _chain / _lanes / _format, emu_process_logs or
// emu_process_records.  The grid-stride kernels run on at most 2 CTAs, so that batches of more than 512 (log_format:
// 128) anomalous records take their stride loops; the scratch block, the R-norm scratch and the output start out
// hostile.  Returns 0, or -6 without an alert format or a batch to word.
extern "C" int emu_encode_alerts(EmuHandle* h, uint64_t first_log_id, int64_t first_alert_id, int64_t now, uint8_t* out,
                                 uint64_t out_cap, uint64_t* out_len, uint64_t* n_alerts, int* declined) {
    if (!h->afmt_set || h->last_src == DMA_SRC_NONE) return -6;
    *out_len = 0; *n_alerts = 0; *declined = 0;
    const uint32_t src = h->last_src, anomaly_cap = (uint32_t)h->anoms.size();
    uint64_t n_lines;
    bool over;
    const uint64_t n_flagged = dm_alert_entries(src, h->hdr, h->last_n_records, anomaly_cap, &n_lines, &over);
    if (over) { *n_alerts = n_flagged; *declined = 1; return 0; }
    if (n_flagged == 0) return 0;
    const uint32_t entries = (uint32_t)n_flagged;
    DmAlertArgs a;
    unsigned long long* tile_sums;
    std::vector<uint8_t> scratch(dm_alert_scratch(nullptr, h->max_lines, anomaly_cap, nullptr, nullptr), 0xEE);
    dm_alert_scratch(scratch.data(), h->max_lines, anomaly_cap, &a, &tile_sums);
    DmAlertHeader ah;
    memset(&ah, 0, sizeof(ah));                                          // as dm_encode_alerts' cudaMemsetAsync of d_ahdr,
    memset(a.rank, 0, n_lines * 4);                                      //   of the ranks
    memset(a.rec_mask, 0, (uint64_t)entries * 4);                        //   and of the merged masks
    std::vector<uint8_t> nbuf(h->msg_bytes + 256, 0xA5), dout(out_cap + 1, 0xEE);
    a.fmt = &h->afmt; a.buf = h->msg; a.nbytes = h->msg_bytes; a.scores = h->last_scores;
    a.anoms = h->anoms.data(); a.n_entries = entries; a.n_lines = n_lines;
    a.ahdr = &ah; a.first_log_id = first_log_id; a.first_alert_id = first_alert_id; a.now = now;
    a.out = dout.data(); a.out_cap = out_cap;
    a.efmt = &h->efmt; a.nbuf = nbuf.data();
    a.src = src;
    if (src == DMA_LOGS) {
        float* rscores;
        uint8_t* rflags;
        const DmLogsArgs la = dm_logs_carve(h->logs.data(), h->logs_cap, h->logs_chunks, &h->lhdr, &rscores, &rflags);
        a.pay = h->in.data(); a.pay_off = la.rec_off; a.pay_len = la.rec_len;
        a.log_line = la.rec_line; a.log_dst = la.line_dst;
    } else if (src == DMA_RECORDS) {
        a.pay = h->in.data(); a.pay_off = h->vals.data(); a.pay_len = h->vals.data() + n_lines;
        a.scores = h->scores.data(); a.flags = h->flags.data(); a.masks = h->masks.data(); a.mons = &h->mons;
    }
    bool fmtl;
    uint64_t mark_n;
    const DmAlertKernel k_mark = dm_alert_mark_kernel(src, false, n_lines, entries, &mark_n);
    const DmAlertKernel k_gather = dm_alert_mark_kernel(src, true, n_lines, entries, &mark_n);
    const DmAlertKernel k_size = dm_alert_pass_kernel(src, h->fmt_set, dm_format_norm(h->fmt), false, &fmtl);
    const DmAlertKernel k_write = dm_alert_pass_kernel(src, h->fmt_set, dm_format_norm(h->fmt), true, &fmtl);
    const unsigned threads = fmtl ? DM_FMTL_THREADS : DMA_THREADS;
    const unsigned mgrid = dm_grid(mark_n, DMA_THREADS, 2), pgrid = dm_grid(entries, threads, 2);
    auto pass = [&](DmAlertKernel k) {
        g_emu_dyn_smem.assign((size_t)2 * h->efmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
        emu_launch_grid(pgrid, threads, [&] { k(a); });
    };
    emu_launch_grid(mgrid, DMA_THREADS, [&] { k_mark(a); });
    emu_scan<uint32_t>(a.rank, n_lines, (uint32_t*)tile_sums, &ah.n_alerts);
    emu_launch_grid(mgrid, DMA_THREADS, [&] { k_gather(a); });
    pass(k_size);
    emu_scan<unsigned long long>(a.size, entries, tile_sums, &ah.total);
    pass(k_write);
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

// The device's Time conversion of the UTF-8 of a str (a ParserSchema Time): 1 and *ts = int(float(s)), or `now` where
// float() must raise ValueError; 0 (declined) otherwise.
extern "C" int emu_alert_time_str(const uint8_t* s, uint32_t n, long long now, long long* ts) {
    return dma_time(s, n, now, ts, true) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------- the MatcherParser stage
// as dm_set_parser_format, on the format of emu_set_format (set with no monitors); nullptr or the reason it refuses
extern "C" const char* emu_set_parser_format(EmuHandle* h, uint32_t n_strings, const uint8_t* strings, const uint32_t* lens,
                                             const uint32_t* capture_order) {
    if (!h->fmt_set) return "emu_set_format has not been called";
    DmParseFmt* P = new DmParseFmt;
    const char* why = dm_parse_fmt_build(h->fmt, n_strings, strings, lens, capture_order, P);
    if (!why) {
        h->pf = *P;
        dm_parse_efmt_build(h->fmt, &h->pfmt);
        h->parse_set = true;
    }
    delete P;
    return why;
}

// As dm_parse_logs: the unwrap without the text copy (walk on at most 2 CTAs), the size pass, the scan and the write
// pass, the parse kernels on at most 2 CTAs so that batches of more than 128 records take their stride loops; the
// scratch, the R-norm scratch and the output start out hostile.  out: out_cap bytes.  Returns 0; -1 for a framing
// error, -6 without a parser format since the last emu_set_format, -4 when the output exceeds out_cap (*out_len then
// tells how large).
extern "C" int emu_parse_logs(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, int delimited, int64_t first_id, int64_t now,
                              uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_records, uint64_t* n_emitted) {
    if (!h->parse_set) return -6;
    const DmFrames fr = dm_frame_records(msg, nbytes, delimited != 0);
    if (fr.error) return -1;
    const uint32_t n = (uint32_t)fr.off.size();
    h->last_src = DMA_SRC_NONE;                                          // (the handle's input is no detected batch)
    DmLogsArgs la;
    float* rscores;
    uint8_t* rflags;
    emu_unwrap(h, msg, nbytes, fr, 0, 2, 0, nullptr, 0, &la, &rscores, &rflags);
    std::vector<uint8_t> nbuf(nbytes + 256, 0xA5), dout(out_cap + 1, 0xEE);
    DmParseArgs a = dm_parse_args(la, &h->pf, &h->pfmt, nbuf.data(), first_id, now);
    unsigned long long *tile_sums, *total;
    std::vector<unsigned long long> scratch(dm_parse_scratch(nullptr, n, nullptr, nullptr, nullptr), 0xDEADBEEFull);
    dm_parse_scratch(scratch.data(), n, &a, &tile_sums, &total);
    *total = 0;                                                          // as dm_parse_logs' cudaMemsetAsync of the total
    const bool norm = dm_format_norm(h->fmt);
    const unsigned grid = dm_grid(n, DM_FMTL_THREADS, 2);
    auto pass = [&](bool write) {
        g_emu_dyn_smem.assign((size_t)2 * h->pfmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
        const DmParseKernel k = dm_parse_kernel(norm, write);
        emu_launch_grid(grid, DM_FMTL_THREADS, [&] { k(a); });
    };
    if (n) {
        pass(false);
        emu_scan<unsigned long long>(a.size, n, tile_sums, total);
    }
    *out_len = *total;
    *n_records = n;
    *n_emitted = h->lhdr.n_lines;
    if (*total > out_cap) return -4;
    if (*total) {
        a.out = dout.data(); a.out_cap = out_cap;
        pass(true);
    }
    memcpy(out, dout.data(), *total);
    return 0;
}

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

// as dm_export_known: every key of the table (own records, peers, emu_import_known), sorted; their count
extern "C" uint64_t emu_export_known(EmuHandle* h, unsigned long long* out, uint64_t cap) {
    std::vector<unsigned long long> v;
    for (unsigned long long k : h->slots)
        if (k) v.push_back(k);
    std::sort(v.begin(), v.end());
    for (uint64_t i = 0; i < v.size() && i < cap; ++i) out[i] = v[i];
    return v.size();
}

// as dm_import_known (dm_k_insert_keys on 2 CTAs of 32 threads); the error bits
extern "C" uint32_t emu_import_known(EmuHandle* h, const unsigned long long* keys, uint64_t n) {
    unsigned int err = 0;
    if (n) emu_launch_grid(2, 32, [&] { dm_k_insert_keys(h->table, keys, n, &err); });
    return err;
}

// ---------------------------------------------------------------------------------------------- window exchange
// As dm_window_words / dm_window_export / dm_window_import / dm_window_pending_keys with seg_keys keys per rank segment
// (libdmdetect: DM_WINDOW_KEYS).  The kernels run on 2 CTAs of 32 threads, so that both take their stride loops.
extern "C" uint64_t emu_window_words(uint32_t world, int with_keys, uint64_t seg_keys) {
    return dm_window_n_words(world, with_keys != 0, seg_keys);
}

extern "C" void emu_window_export(EmuHandle* h, unsigned long long* buf, uint32_t rank, uint32_t world, int with_keys,
                                  uint64_t seg_keys) {
    DmWindowKeys wk{h->novel_exported, h->novel_exported, 0};
    if (with_keys) {
        wk = dm_window_keys(h->novel_exported, h->counts[1], h->table.novel_cap, seg_keys);
        h->novel_pending = wk.pending;
    }
    const uint64_t n_words = dm_window_n_words(world, with_keys != 0, seg_keys);
    const uint64_t seg_off = dm_window_n_words(rank, true, seg_keys);
    emu_launch_grid(2, 32, [&] {
        dm_k_window_export(buf, n_words, h->stats, h->stats_exported, h->novel.data(), wk.from, wk.to, seg_off, seg_keys,
                           with_keys);
    });
    h->novel_exported = wk.to;
}

extern "C" uint64_t emu_window_pending_keys(EmuHandle* h) { return h->novel_pending; }

// the error bits the import leaves in the handle's error word (dm_sync reports them)
extern "C" uint32_t emu_window_import(EmuHandle* h, const unsigned long long* buf, uint32_t rank, uint32_t world,
                                      int with_keys, uint64_t seg_keys) {
    unsigned int err = 0;
    emu_launch_grid(2, 32, [&] {
        dm_k_window_import(buf, world, rank, seg_keys, h->stats_global, h->table, &err, with_keys);
    });
    return err;
}

extern "C" void emu_get_global_stats(EmuHandle* h, unsigned long long* out) {
    for (int i = 0; i < DM_STATS_WORDS; ++i) out[i] = h->stats_global[i];
}
