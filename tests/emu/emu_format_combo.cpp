// emu_format_combo.cpp -- the emulator of emu_tile.cpp plus log_format mode WITH combination monitors: the COMBO
// instantiations of dm_k_format_lanes, launched as dm_process_lines launches them when dm_set_combos has set
// combinations.  TEST INFRASTRUCTURE ONLY: built by tests/test_format_combos.py into tests/emu/_build/; never part of
// libdmdetect.so.  It includes emu_tile.cpp whole (its runtime, handle and emu_set_format / emu_set_combos state), so
// this library exports every emu_* function of emu_tile.cpp as well.
#include "emu_tile.cpp"

// Mirrors the fmt branch of dm_process_lines with combinations set (emu_set_combos): K_A (dm_k_rowindex) writes the
// record index and the batch header, then the train / detect launches of dm_k_format_lanes<TRAIN, NORM, true> on a
// 3-CTA grid, so that messages of more than 192 records take the kernel's stride loop.  Without combinations it runs
// the single-monitor instantiations, as the library does.  Hostile slack as in emu_process_format.
extern "C" int emu_process_format_combo(EmuHandle* h, const uint8_t* msg, uint64_t nbytes, uint64_t n_train, uint8_t* flags,
                                        float* scores, uint64_t cap, uint64_t* n_lines, uint64_t* n_anoms, uint32_t* err) {
    if (!g_fmt_set) return -6;
    *n_lines = 0; *n_anoms = 0; *err = 0;
    if (nbytes == 0) { memset(&h->hdr, 0, sizeof(h->hdr)); return 0; }      // as dm_process_lines: no launch at all
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
    a.stats = h->stats; a.nbytes = nbytes;
    static DmMonitors cm;                                      // combination monitors (emu_set_combos), as dm_set_combos leaves them
    memset(&cm, 0, sizeof(cm));
    cm.n = g_fmt.n_mons; cm.n_combos = g_n_combos; cm.member_only = g_member_only;
    for (size_t i = 0; i < g_combo_off.size(); ++i) cm.combo_off[i] = g_combo_off[i];
    for (size_t i = 0; i < g_combo_members.size(); ++i) cm.combo_members[i] = (uint8_t)g_combo_members[i];
    const bool combo = g_n_combos > 0;
    a.combos = combo ? &cm : nullptr;
    g_emu_dyn_smem.assign((size_t)2 * g_fmt.max_slots * DM_FMTL_THREADS * sizeof(uint2), 0xEE);
    const bool norm = g_fmt.norm_flags != 0 && g_fmt.n_chains > 1;
    uint8_t* nbuf = (uint8_t*)aligned_alloc(64, ((nbytes + 256 + 63) / 64) * 64);
    memset(nbuf, 0xA5, nbytes + 256);
    if (n_train > 0) {
        a.line_lo = 0; a.line_hi = n_train;
        if (combo && norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, true, true>(a, &g_fmt, nbuf); });
        else if (combo) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, false, true>(a, &g_fmt, nbuf); });
        else if (norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, true, false>(a, &g_fmt, nbuf); });
        else emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<true, false, false>(a, &g_fmt, nbuf); });
    }
    a.line_lo = n_train; a.line_hi = ~0ull;
    if (combo && norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, true, true>(a, &g_fmt, nbuf); });
    else if (combo) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, false, true>(a, &g_fmt, nbuf); });
    else if (norm) emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, true, false>(a, &g_fmt, nbuf); });
    else emu_launch_grid(3, DM_FMTL_THREADS, [&] { dm_k_format_lanes<false, false, false>(a, &g_fmt, nbuf); });
    free(nbuf);
    free(buf);
    *n_lines = h->hdr.n_lines;
    *n_anoms = h->hdr.n_anomalies;
    *err = h->hdr.error;
    return 0;
}
