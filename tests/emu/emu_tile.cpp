// emu_tile.cpp -- runs the product's kernel sources (dm_kernels_*.cuh) on the CPU
// emulator.  TEST INFRASTRUCTURE ONLY: built by tests/emu/build.py into tests/emu/_build/,
// loaded by tests/test_emu_tile.py; never part of libdmdetect.so.
#include "cuda_emu.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "dm_kernels_index.cuh"
#include "dm_kernels_stream.cuh"
#include "dm_kernels_records.cuh"
#include "dm_kernels_format.cuh"
#include "dm_kernels_lanes.cuh"
#include "dm_format_host.h"

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

struct EmuHandle {
    DmKeys keys;
    DmTable table;
    std::vector<unsigned long long> slots, novel;
    unsigned long long counts[2] = {0, 0};
    unsigned long long stats[DM_STATS_WORDS] = {0};
    DmBatchHeader hdr;
    std::vector<dm_anomaly_t> anoms;
    uint64_t max_lines = 0;
    // rows variant
    std::vector<uint32_t> row_prefix;
    std::vector<unsigned long long> rows_tile_state;
    unsigned long long row_ctr = 0, row_ctr_base = 0;
    uint32_t rows_epoch = 0;
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

// Mirrors dmx_launch (dm_kernels_stream.cuh): [row counts, boundary, TRAIN launch,] DETECT launch.  The grid is
// `g_emu_stream_ctas` CTAs run one after the other (the last one runs the epilogue).
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
    uint8_t* buf = (uint8_t*)aligned_alloc(64, ((nbytes + 64 + 63) / 64) * 64 + 64);
    memcpy(buf, msg, nbytes);
    for (int i = 0; i < 64; ++i) buf[nbytes + i] = (i & 1) ? '\n' : '=';      // hostile slack
    // as dm_process_lines: the header is the previous call's until this call's epilogue rewrites it (its take-out of
    // the previous call's alerts reads it), except for an empty message; errors are read as dm_sync reads them
    *n_lines = 0; *n_anoms = 0; *err = 0;
    const uint32_t n_rows = (uint32_t)((nbytes + DMX_ROW - 1) / DMX_ROW);
    if (n_rows == 0) {
        memset(&h->hdr, 0, sizeof(h->hdr));
        *err = g_xs.sh.error;
        g_xs.sh.error = 0;
        free(buf);
        return 0;
    }
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
    const unsigned long long warps_max = (unsigned long long)g_emu_stream_ctas * DMX_WARPS;
    const uint32_t rpw = (uint32_t)((n_rows + warps_max - 1) / warps_max);
    const unsigned long long warps = (n_rows + rpw - 1) / rpw;
    const unsigned grid = (unsigned)((warps + DMX_WARPS - 1) / DMX_WARPS);
    a.rows_per_warp = rpw;
    a.rows_per_cta = rpw * DMX_WARPS;
    a.ctas_per_grp = (grid + DMX_THREADS - 1) / DMX_THREADS;
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

// Record mode on the device: mirrors dm_process_records (framing walk on the host, then
// dm_k_records train pass + detect pass).  `mons` uses the dm_monitor_t layout.
static uint32_t g_n_combos = 0, g_member_only = 0;
static std::vector<uint32_t> g_combo_off, g_combo_members;
// mirrors dm_set_combos; applies to the following emu_process_records calls (0 combos = off)
extern "C" void emu_set_combos(uint32_t n_combos, const uint32_t* member_off, const uint32_t* members, uint32_t member_only) {
    g_n_combos = n_combos;
    g_member_only = member_only;
    g_combo_off.assign(member_off, member_off + (n_combos ? n_combos + 1 : 0));
    g_combo_members.assign(members, members + (n_combos ? member_off[n_combos] : 0));
}

extern "C" int emu_process_records(EmuHandle* h, const DmMonitor* mons, uint32_t n_mons, const uint8_t* msg,
                                   uint64_t nbytes, uint32_t n_train, uint8_t* flags, float* scores, uint32_t* masks,
                                   uint64_t cap, uint64_t* n_records, uint64_t* n_anoms) {
    static DmMonitors hm;
    memset(&hm, 0, sizeof(hm));
    hm.n = n_mons;
    for (uint32_t i = 0; i < n_mons; ++i) hm.m[i] = mons[i];
    hm.n_combos = g_n_combos;
    hm.member_only = g_member_only;
    for (size_t i = 0; i < g_combo_off.size(); ++i) hm.combo_off[i] = g_combo_off[i];
    for (size_t i = 0; i < g_combo_members.size(); ++i) hm.combo_members[i] = (uint8_t)g_combo_members[i];
    std::vector<uint32_t> off, len;
    uint64_t pos = 0;
    while (pos < nbytes) {
        uint64_t l = 0; int shift = 0;
        for (;;) {
            if (pos >= nbytes) return -1;
            const uint8_t b = msg[pos++];
            l |= (uint64_t)(b & 0x7F) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (l > nbytes - pos) return -1;
        off.push_back((uint32_t)pos); len.push_back((uint32_t)l);
        pos += l;
    }
    const uint32_t n = (uint32_t)off.size();
    if (n > cap) return -4;
    memset(&h->hdr, 0, sizeof(h->hdr));
    DmRecordsArgs a;
    a.buf = msg; a.rec_off = off.data(); a.rec_len = len.data(); a.n_records = n; a.n_train_records = n_train;
    a.mons = &hm; a.table = h->table; a.flags = flags; a.scores = scores; a.masks = masks; a.hdr = &h->hdr; a.stats = h->stats;
    uint32_t bound[2] = {0, 0};
    if (n) {
        if (n_train > 0) {
            emu_launch(128, [&] { dm_k_records(a, 2); });
            emu_launch(256, [&] { dm_k_records_bound(flags, n, n_train, bound); });
            emu_launch(128, [&] { dm_k_records(a, 0, bound); });
        }
        if (n_train < n) emu_launch(128, [&] { dm_k_records(a, 1, n_train > 0 ? bound : nullptr); });
    }
    h->stats[0] += n;
    h->stats[1] += bound[1];
    h->stats[2] += n - (n_train > 0 ? bound[0] : 0);
    *n_records = n;
    *n_anoms = h->hdr.n_anomalies;
    return 0;
}

extern "C" void emu_chain_stats(unsigned long long* out, int reset) {
    for (int i = 0; i < 8; ++i) { out[i] = g_emu_chain_stats[i]; if (reset) g_emu_chain_stats[i] = 0; }
}

// log_format / template mode: mirrors dm_set_format + the fmt branch of dm_process_lines: K_A (dm_k_rowindex) writes the
// record index and the batch header, then the train / detect launches of dm_k_format_lanes on a 3-CTA grid, so that
// messages of more than 192 records take the kernel's stride loop.
static DmFormat g_fmt;
static bool g_fmt_set = false;
static char g_fmt_err[256];
extern "C" const char* emu_set_format(const DmMonitor* mons, uint32_t n_mons, const char* log_format, const char* content_name,
                                      uint32_t n_templates, const char* const* templates, uint32_t norm_flags) {
    static DmMonitors hm;
    memset(&hm, 0, sizeof(hm));
    hm.n = n_mons;
    for (uint32_t i = 0; i < n_mons; ++i) hm.m[i] = mons[i];
    std::string err;
    g_fmt_set = dm_format_build(log_format, content_name, n_templates, templates, norm_flags, hm, &g_fmt, &err);
    snprintf(g_fmt_err, sizeof(g_fmt_err), "%s", err.c_str());
    return g_fmt_set ? nullptr : g_fmt_err;
}

extern "C" int emu_process_format(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                  float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    if (!g_fmt_set) return -6;
    *n_lines = 0; *n_anoms = 0; *err = 0;
    if (nbytes == 0) { memset(&h->hdr, 0, sizeof(h->hdr)); return 0; }      // as dm_process_lines: no launch at all
    // hostile slack: the bytes of the configured literals, each followed by '\n', over and over (the kernel reads up to
    // 12 bytes past a record; none of it may count)
    std::vector<uint8_t> lit_bytes;
    for (uint32_t i = 0; i < g_fmt.chain_first[g_fmt.n_chains]; ++i) {
        for (uint32_t j = 0; j < g_fmt.lit_len[i]; ++j) lit_bytes.push_back((uint8_t)(g_fmt.pool[g_fmt.lit_off[i] + j / 4] >> (8 * (j % 4))));
        lit_bytes.push_back('\n');
    }
    uint8_t* buf = (uint8_t*)aligned_alloc(64, ((nbytes + 64 + 63) / 64) * 64 + 64);
    memcpy(buf, msg, nbytes);
    for (uint32_t i = 0; i < 64; ++i) buf[nbytes + i] = lit_bytes[i % lit_bytes.size()];
    const uint32_t n_rows = (uint32_t)((nbytes + DMR_ROW - 1) / DMR_ROW);
    DmRowsArgs ra;
    ra.buf = buf; ra.nbytes = nbytes; ra.n_rows = n_rows; ra.n_tiles = (n_rows + DMR_TILE_ROWS - 1) / DMR_TILE_ROWS;
    h->row_prefix.assign(n_rows + 1, 0xDEADBEEFu);
    if (h->rows_tile_state.size() < ra.n_tiles + 1) h->rows_tile_state.resize(ra.n_tiles + 1, 0);
    ra.row_prefix = h->row_prefix.data(); ra.tile_state = h->rows_tile_state.data();
    h->rows_epoch = (h->rows_epoch % 0x3FFFFFFEu) + 1u;
    ra.epoch = h->rows_epoch;
    ra.keys = &h->keys; ra.table = h->table; ra.flags = flags; ra.scores = scores; ra.out_cap = cap;
    ra.anomalies = h->anoms.data(); ra.anomaly_cap = (uint32_t)h->anoms.size(); ra.hdr = &h->hdr; ra.stats = h->stats;
    ra.row_ctr = &h->row_ctr; ra.n_train_lines = n_train; ra.max_lines = h->max_lines;
    ra.line_lo = 0; ra.line_hi = ~0ull; ra.ctr_base = h->row_ctr_base; ra.aux_counts = nullptr;
    std::vector<uint32_t> ls(h->max_lines + 2, 0xDEADBEEFu);
    ra.line_start = ls.data(); ra.group = DMR_GROUP; ra.static_rows = 0; ra.timeline = nullptr;
    emu_launch_grid(ra.n_tiles, DMR_A_THREADS, [&] { dm_k_rowindex(ra); });
    DmDetectArgs a;
    a.buf = buf; a.line_start = ls.data(); a.hdr_in = &h->hdr; a.hdr = &h->hdr; a.keys = &h->keys; a.table = h->table;
    a.flags = flags; a.scores = scores; a.out_cap = cap; a.anomalies = h->anoms.data(); a.anomaly_cap = (uint32_t)h->anoms.size();
    a.stats = h->stats; a.combos = nullptr; a.nbytes = nbytes;
    g_emu_dyn_smem.assign((size_t)2 * g_fmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
    // R-norm scratch: hostile content (the kernel may only read back what it wrote itself)
    const bool norm = g_fmt.norm_flags != 0 && g_fmt.n_chains > 1;
    uint8_t* nbuf = (uint8_t*)aligned_alloc(64, ((nbytes + 256 + 63) / 64) * 64);
    memset(nbuf, 0xA5, nbytes + 256);
    // the launches of dm_process_lines; a CTA whose first record is past the record count (or a header error) leaves
    if (n_train > 0) {
        a.line_lo = 0; a.line_hi = n_train;
        if (norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, true>(a, &g_fmt, nbuf); });
        else emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, false>(a, &g_fmt, nbuf); });
    }
    a.line_lo = n_train; a.line_hi = ~0ull;
    if (norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, true>(a, &g_fmt, nbuf); });
    else emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, false>(a, &g_fmt, nbuf); });
    free(nbuf);
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error;
    return 0;
}

// one thread per record (dm_kernels_lanes.cuh): K_A writes the record index, as in dm_lanes_launch
extern "C" int emu_process_lanes(EmuHandle* h, const uint8_t* msg_in, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                 float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    uint8_t* buf = (uint8_t*)aligned_alloc(64, ((nbytes + 64 + 63) / 64) * 64 + 64);
    memcpy(buf, msg_in, nbytes);
    for (int i = 0; i < 64; ++i) buf[nbytes + i] = (i & 1) ? '\n' : '=';      // hostile slack
    memset(&h->hdr, 0, sizeof(h->hdr));
    *n_lines = 0; *n_anoms = 0; *err = 0;
    const uint32_t n_rows = (uint32_t)((nbytes + DMR_ROW - 1) / DMR_ROW);
    if (n_rows == 0) { free(buf); return 0; }
    DmRowsArgs ra;
    ra.buf = buf; ra.nbytes = nbytes; ra.n_rows = n_rows; ra.n_tiles = (n_rows + DMR_TILE_ROWS - 1) / DMR_TILE_ROWS;
    h->row_prefix.assign(n_rows + 1, 0xDEADBEEFu);
    if (h->rows_tile_state.size() < ra.n_tiles + 1) h->rows_tile_state.resize(ra.n_tiles + 1, 0);
    ra.row_prefix = h->row_prefix.data(); ra.tile_state = h->rows_tile_state.data();
    h->rows_epoch = (h->rows_epoch % 0x3FFFFFFEu) + 1u;
    ra.epoch = h->rows_epoch;
    ra.keys = &h->keys; ra.table = h->table; ra.flags = flags; ra.scores = scores; ra.out_cap = cap;
    ra.anomalies = h->anoms.data(); ra.anomaly_cap = (uint32_t)h->anoms.size(); ra.hdr = &h->hdr; ra.stats = h->stats;
    ra.row_ctr = &h->row_ctr; ra.n_train_lines = n_train; ra.max_lines = h->max_lines;
    ra.line_lo = 0; ra.line_hi = ~0ull; ra.ctr_base = h->row_ctr_base; ra.aux_counts = nullptr;
    std::vector<uint32_t> ls(h->max_lines + 2, 0xDEADBEEFu);
    ra.line_start = ls.data(); ra.group = DMR_GROUP; ra.static_rows = 0; ra.timeline = nullptr;
    emu_launch_grid(ra.n_tiles, DMR_A_THREADS, [&] { dm_k_rowindex(ra); });
    const uint64_t n = h->hdr.n_lines;
    if (h->hdr.error == 0 && n <= cap) {
        DmDetectArgs a;
        a.buf = buf; a.line_start = ls.data(); a.hdr_in = &h->hdr; a.hdr = &h->hdr; a.keys = &h->keys; a.table = h->table;
        a.flags = flags; a.scores = scores; a.out_cap = cap; a.anomalies = h->anoms.data(); a.anomaly_cap = (uint32_t)h->anoms.size();
        a.stats = h->stats; a.nbytes = nbytes;
        const uint64_t nt = std::min<uint64_t>(n_train, n);
        const unsigned blocks = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + DM_LANES_THREADS - 1) / DM_LANES_THREADS, 5));
        static DmMonitors cm;                                  // combination monitors (emu_set_combos), as dm_set_combos leaves them
        memset(&cm, 0, sizeof(cm));
        cm.n = h->keys.n; cm.n_combos = g_n_combos; cm.member_only = g_member_only;
        for (size_t i = 0; i < g_combo_off.size(); ++i) cm.combo_off[i] = g_combo_off[i];
        for (size_t i = 0; i < g_combo_members.size(); ++i) cm.combo_members[i] = (uint8_t)g_combo_members[i];
        a.combos = g_n_combos ? &cm : nullptr;
        g_emu_dyn_smem.assign((size_t)DM_MAX_KEYS * DM_LANES_THREADS * sizeof(unsigned long long), 0);
        if (g_n_combos) {
            if (nt > 0) { a.line_lo = 0; a.line_hi = nt; emu_launch_grid(blocks, DM_LANES_THREADS, [&] { dm_k_lanes<true, true>(a); }); }
            if (nt < n) { a.line_lo = nt; a.line_hi = ~0ull; emu_launch_grid(blocks, DM_LANES_THREADS, [&] { dm_k_lanes<false, true>(a); }); }
        } else {
            if (nt > 0) { a.line_lo = 0; a.line_hi = nt; emu_launch_grid(blocks, DM_LANES_THREADS, [&] { dm_k_lanes<true, false>(a); }); }
            if (nt < n) { a.line_lo = nt; a.line_hi = ~0ull; emu_launch_grid(blocks, DM_LANES_THREADS, [&] { dm_k_lanes<false, false>(a); }); }
        }
    }
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error;
    return 0;
}

extern "C" uint32_t emu_get_anomalies(EmuHandle* h, dm_anomaly_t* out, uint32_t cap) {
    uint32_t n = std::min<uint32_t>(h->hdr.anomaly_list_count, (uint32_t)h->anoms.size());
    std::vector<dm_anomaly_t> v(h->anoms.begin(), h->anoms.begin() + n);
    std::sort(v.begin(), v.end(), [](const dm_anomaly_t& a, const dm_anomaly_t& b) { return a.line < b.line; });
    uint32_t m = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (m && out[m - 1].line == v[i].line) { out[m - 1].mask |= v[i].mask; continue; }
        if (m >= cap) break;
        out[m++] = v[i];
    }
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
