// dm_kernels_lanes.cuh -- key=value tokenizer + detector with ONE THREAD PER RECORD.
//
// The other variants spread the bytes of a record over the lanes of a warp and pay for it
// with queues, ballots and partially filled passes (rows: ~340 warp instructions per 256-byte
// record, 19 of 32 lanes active).  Here every lane walks its own record as a small state
// machine over 4-byte words (R-tok L2-L6 kept exactly: quote parity, field starts, the first
// '=' of a field), records the '=' whose key can be a monitored one in a per-lane queue, and
// afterwards identifies / hashes / probes its queue in position order -- the lanes of a warp
// run that second phase in lockstep over the queue index, so nothing serialises.  No warp
// collectives at all; reads go through L1 (a lane streams through its record, every 32-byte
// sector is used by eight consecutive word loads), outputs are written one record per lane,
// i.e. coalesced.
//
// What it replaces: per record, MatcherParser (fields) + NewValueDetector.train / .detect from
// the un-vendored detectmatelibrary, driven by /root/reference/src/service/core.py:201-203.
// Needs the line index (dm_kernels_index.cuh K_A).  Rules: DESIGN.md R-tok, R-spec 1-4.
#pragma once
#include "dm_device.cuh"
#include "dm_kernels_index.cuh"     // K_A (dm_k_rowindex) writes the record index
#include "dm_kernels_records.cuh"   // DmMonitors: combination monitors (dm_set_combos)

#define DM_LANES_THREADS 64         // small CTAs: a 64k-record message is only 2048 warps, spread them evenly
#define DM_LANES_Q 20               // queued '=' per record before the queue is drained early

// 0x80 in every byte of x that is zero
__device__ __forceinline__ uint32_t dm_zeroflags(uint32_t x) {
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}

// 4-bit mask of the bytes of w in 0x20..0x27 or equal to '='
__device__ __forceinline__ uint32_t dm_lanes_cand(uint32_t w) {
    return dm_flags_to_nib(dm_zeroflags((w & 0xF8F8F8F8u) ^ 0x20202020u) | dm_eqflags(w, 0x3D3D3D3Du));
}

// COMBO: the record's value fingerprints are kept (fps[k * DM_LANES_THREADS], this lane's column) for
// the combination monitors evaluated after the record; member-only fields do not alert themselves.
template <bool TRAIN, bool COMBO>
__device__ __forceinline__ void dm_lanes_event(const DmDetectArgs& a, const DmKeys& sk, uint32_t q, uint32_t& seen,
                                               uint32_t& unknown, unsigned long long* fps, uint32_t member_only) {
    const int k = dm_key_identify(a.buf, q, sk);
    if (k < 0 || ((seen >> k) & 1u)) return;                       // not monitored / not the first occurrence (L6)
    seen |= 1u << k;
    const uint64_t fp = dm_hash_value(a.buf, a.nbytes, (uint64_t)q + 1);
    if (COMBO) {
        fps[(uint32_t)k * DM_LANES_THREADS] = fp;
        if ((member_only >> k) & 1u) return;
    }
    const uint64_t key = dm_make_key(fp, sk.salt[k]);
    if (TRAIN) dm_table_insert(a.table, key, &a.hdr->error);
    else if (!dm_table_contains(a.table, key)) unknown |= 1u << k;
}

template <bool TRAIN, bool COMBO>
__global__ void __launch_bounds__(DM_LANES_THREADS) dm_k_lanes(DmDetectArgs a) {
#ifdef DM_EMU
    unsigned long long* s_fp = reinterpret_cast<unsigned long long*>(g_emu_dyn_smem.data());
#else
    extern __shared__ unsigned long long s_fp[];                  // COMBO: [n_keys][DM_LANES_THREADS] value fingerprints
#endif
    __shared__ DmKeys sk;
    __shared__ uint32_t s_q[DM_LANES_Q][DM_LANES_THREADS];
    __shared__ unsigned int s_unk[DM_MAX_KEYS];
    __shared__ unsigned long long s_anom, s_score;
    dm_pdl_wait();                                                // K_A / the training pass are complete (dm_kernels_index.cuh)
    {
        // CTAs without records (the grid is sized for the worst case) leave before touching anything
        const uint64_t n_lines0 = a.hdr_in->n_lines;
        const uint64_t hi0 = a.line_hi < n_lines0 ? a.line_hi : n_lines0;
        if (a.hdr_in->error || a.line_lo + (uint64_t)blockIdx.x * blockDim.x >= hi0) return;
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(a.keys);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sk);
        for (uint32_t i = threadIdx.x; i < sizeof(DmKeys) / 4; i += blockDim.x) dst[i] = src[i];
        if (threadIdx.x < DM_MAX_KEYS) s_unk[threadIdx.x] = 0;
        if (threadIdx.x == 0) { s_anom = 0; s_score = 0; }
    }
    __syncthreads();
    unsigned long long lenmask = 0;                               // bit L: some monitored key has length L
    for (uint32_t k = 0; k < sk.n; ++k) lenmask |= 1ull << sk.len[k];

    if (a.hdr_in->error) return;                                  // K_A: more records than the index / outputs hold
    const uint8_t* __restrict__ buf = a.buf;
    const uint32_t tid = threadIdx.x;
    const DmMonitors* __restrict__ cm = reinterpret_cast<const DmMonitors*>(a.combos);
    const uint32_t member_only = COMBO ? cm->member_only : 0u;
    const uint64_t n_lines = a.hdr_in->n_lines;
    const uint64_t hi = a.line_hi < n_lines ? a.line_hi : n_lines;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;

    for (uint64_t line = a.line_lo + (uint64_t)blockIdx.x * blockDim.x + tid; line < hi; line += stride) {
        const uint32_t s = a.line_start[line];
        const uint32_t e = a.line_start[line + 1] - 1;             // the '\n' (or nbytes)
        uint32_t cnt = 0, seen = 0, unknown = 0;
        uint32_t inq = 0, kopen = 1, kstart = s;                  // a record starts with a field (L4, p == 0)
        uint4 vnext = make_uint4(0, 0, 0, 0);
        if ((s & ~15u) < e) vnext = __ldg(reinterpret_cast<const uint4*>(buf + (s & ~15u)));
        for (uint32_t p = s & ~15u; p < e; p += 16) {
            const uint4 v = vnext;
            if (p + 16 < e) vnext = __ldg(reinterpret_cast<const uint4*>(buf + p + 16));   // in flight during the state machine
            // candidate bytes: 0x20..0x27 (space " ' among them) and '='; nothing else changes the state.
            // The four words are independent (ILP); the state machine below only visits candidates.
            uint32_t m = dm_lanes_cand(v.x) | (dm_lanes_cand(v.y) << 4) | (dm_lanes_cand(v.z) << 8) | (dm_lanes_cand(v.w) << 12);
            if (p < s) m &= 0xFFFFu << (s - p);
            if (e - p < 16u) m &= (1u << (e - p)) - 1u;
            while (m) {
                const uint32_t b = (uint32_t)__ffs(m) - 1u;
                m &= m - 1;
                const uint32_t wsel = b >> 2;
                const uint32_t w = wsel == 0 ? v.x : (wsel == 1 ? v.y : (wsel == 2 ? v.z : v.w));
                const uint32_t c = (w >> (8u * (b & 3u))) & 0xFFu;
                const uint32_t q = p + b;
                if (c == 0x3Du) {                                  // '=': ends the key of an open field
                    const uint32_t klen = q - kstart;
                    if (kopen && klen >= 1u && klen <= DM_MAX_KEYLEN && ((lenmask >> klen) & 1ull)) {
                        if (cnt == DM_LANES_Q) {                   // rare: drain, keeping position order
                            for (uint32_t j = 0; j < cnt; ++j) dm_lanes_event<TRAIN, COMBO>(a, sk, s_q[j][tid], seen, unknown, s_fp + tid, member_only);
                            cnt = 0;
                        }
                        s_q[cnt++][tid] = q;
                    }
                    kopen = 0;
                } else if (c == 0x20u || c == 0x27u) {             // space or ': a field may start behind it (L4)
                    kopen = inq ^ 1u;
                    kstart = q + 1;
                } else if (c == 0x22u) {                           // '"'
                    inq ^= 1u;
                    kopen = 0;
                }
            }
        }
        for (uint32_t j = 0; j < cnt; ++j) dm_lanes_event<TRAIN, COMBO>(a, sk, s_q[j][tid], seen, unknown, s_fp + tid, member_only);

        if (COMBO) {
            // combination c = ordered tuple of the member fields' values; needs every member present
            const uint32_t n_combos = cm->n_combos;
            for (uint32_t c = 0; c < n_combos; ++c) {
                const uint32_t lo = cm->combo_off[c], hi_m = cm->combo_off[c + 1];
                uint64_t acc = dm_combo_seed(hi_m - lo);
                bool all = true;
                for (uint32_t j = lo; j < hi_m; ++j) {
                    const uint32_t k = cm->combo_members[j];
                    if (!((seen >> k) & 1u)) { all = false; break; }
                    acc = dm_combo_fold(acc, s_fp[k * DM_LANES_THREADS + tid]);
                }
                if (!all) continue;
                const uint64_t key = dm_make_key(acc ? acc : 1ull, dm_field_salt(sk.n + c));
                if (TRAIN) dm_table_insert(a.table, key, &a.hdr->error);
                else if (!dm_table_contains(a.table, key)) unknown |= 1u << (sk.n + c);
            }
        }
        const uint32_t n_unk = (uint32_t)__popc(unknown);
        if (line < a.out_cap) {
            if (a.flags) a.flags[line] = n_unk ? 1 : 0;
            if (a.scores) a.scores[line] = (float)n_unk;
        }
        if (n_unk) {
            atomicAdd(&s_anom, 1ull);
            atomicAdd(&s_score, (unsigned long long)n_unk);
            uint32_t m = unknown;
            while (m) { const int b = __ffs(m) - 1; m &= m - 1; atomicAdd(&s_unk[b], 1u); }
            const unsigned int at = atomicAdd(&a.hdr->anomaly_list_count, 1u);
            if (at < a.anomaly_cap) {
                dm_anomaly_t r; r.line = (uint32_t)line; r.mask = unknown; r.offset = s;
                a.anomalies[at] = r;
            }
        }
    }
    dm_pdl_launch_dependents();                                   // the next step's K_A may start streaming its message in
    __syncthreads();
    if (!TRAIN) {
        if (threadIdx.x == 0 && s_anom) {
            atomicAdd(&a.hdr->n_anomalies, s_anom);
            atomicAdd(&a.stats[3], s_anom);
            atomicAdd(&a.stats[4], s_score);
        }
        if (threadIdx.x < DM_MAX_KEYS && s_unk[threadIdx.x])
            atomicAdd(&a.stats[8 + threadIdx.x], (unsigned long long)s_unk[threadIdx.x]);
    }
}

// The instantiation a launch runs.
typedef void (*DmLanesKernel)(DmDetectArgs);
static inline DmLanesKernel dm_lanes_kernel(bool train, bool combo) {
    if (train) return combo ? dm_k_lanes<true, true> : dm_k_lanes<true, false>;
    return combo ? dm_k_lanes<false, true> : dm_k_lanes<false, false>;
}

#ifndef DM_EMU
// K_A (row index + record index) then one thread per record.  Returns the number of launches.
static inline int dm_lanes_launch(DmRowsScratch* s, uint32_t* d_line_start, const uint8_t* d_buf, uint64_t nbytes,
                                  uint64_t n_train_lines, const DmKeys* d_keys, DmTable table, uint8_t* d_flags,
                                  float* d_scores, uint64_t out_cap, dm_anomaly_t* d_anoms, uint32_t anomaly_cap,
                                  DmBatchHeader* d_hdr, unsigned long long* d_stats, uint64_t max_lines, int sm_count,
                                  const void* d_combos, uint32_t n_keys,
                                  cudaStream_t st, void (*mark)(void*, cudaStream_t, int), void* mark_ctx) {
    if ((nbytes + DMR_ROW - 1) / DMR_ROW > s->max_rows) return DM_ERR_CAPACITY;
    const DmRowsArgs ra = dm_rows_args(d_buf, nbytes, s->d_row_prefix, s->d_tile_state, &s->epoch, d_line_start, d_flags,
                                       d_scores, out_cap, d_hdr, d_stats, n_train_lines, max_lines);
    if (ra.n_rows == 0) return 0;
    int launched = 0;
    dm_launch_pdl(dm_k_rowindex, ra.n_tiles, DMR_A_THREADS, st, s->pdl, ra);
    ++launched;
    DmDetectArgs a = dm_detect_args(d_buf, nbytes, d_line_start, d_hdr, d_keys, table, d_flags, d_scores, out_cap, d_anoms,
                                    anomaly_cap, d_stats, d_combos);
    const unsigned grid = dm_detect_grid(nbytes, max_lines, DM_LANES_THREADS, (uint64_t)sm_count * 32);
    // (the record kernels themselves are launched normally: their records sit in the first CTAs of
    // a worst-case grid, and an early launch into whatever slots K_A leaves free places those
    // CTAs unevenly -- measured 2x slower; the next step's K_A still overlaps their tail)
    const size_t smem = d_combos ? (size_t)n_keys * DM_LANES_THREADS * sizeof(unsigned long long) : 0;
    if (n_train_lines > 0) {
        a.line_lo = 0; a.line_hi = n_train_lines;
        dm_launch_pdl_smem(dm_lanes_kernel(true, d_combos != nullptr), grid, DM_LANES_THREADS, smem, st, false, a);
        ++launched;
    }
    a.line_lo = n_train_lines; a.line_hi = ~0ull;
    if (mark) mark(mark_ctx, st, 0);
    dm_launch_pdl_smem(dm_lanes_kernel(false, d_combos != nullptr), grid, DM_LANES_THREADS, smem, st, false, a);
    if (mark) mark(mark_ctx, st, 1);
    ++launched;
    if (cudaGetLastError() != cudaSuccess) return DM_ERR_CUDA;
    return launched;
}
#endif  // DM_EMU
