// dm_kernels_window.cuh -- the multi-GPU window exchange (dm_window_export / dm_window_import), the known-set
// import (dm_import_known) and export (dm_export_known).
//
// Buffer layout (uint64 words): [0, DM_STATS_WORDS) the statistics delta, summed over ranks; with keys, then per rank r
// a segment [count, key_0 .. key_{seg_keys-1}] that only rank r fills, so the SUM all-reduce concatenates the
// segments.  libdmdetect passes seg_keys = DM_WINDOW_KEYS; the host side of an export is dm_window_keys (dm_host.h).
#pragma once
#include "dm_device.cuh"
#include "dm_kernels_alerts.cuh"     // the exclusive scan (dm_k_alert_scan_*) the export's digit offsets go through

// The words of a window buffer of `world` ranks with seg_keys keys per rank segment.
inline uint64_t dm_window_n_words(uint32_t world, bool with_keys, uint64_t seg_keys) {
    return (uint64_t)DM_STATS_WORDS + (with_keys ? (uint64_t)world * (1ull + seg_keys) : 0ull);
}

// This rank's part of a window: the statistics delta since the previous export (word 6, the known-key count, travels as
// 0: each rank's table count already holds the keys of every rank) and, with keys, novel[novel_from, novel_to) in its
// segment at seg_off.  Every other word is written 0.
__global__ void dm_k_window_export(unsigned long long* __restrict__ out, uint64_t n_words,
                                   unsigned long long* __restrict__ stats, unsigned long long* __restrict__ exported,
                                   const unsigned long long* __restrict__ novel, uint64_t novel_from, uint64_t novel_to,
                                   uint64_t seg_off, uint64_t seg_keys, int with_keys) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = tid; i < n_words; i += nth) {
        unsigned long long v = 0;
        if (i < DM_STATS_WORDS) {
            unsigned long long cur = (i == 6) ? 0ull : stats[i];
            v = cur - atomicExch(exported + i, cur);      // telescopes mod 2^64 whatever the order of in-flight windows
        } else if (with_keys && i >= seg_off && i < seg_off + 1 + seg_keys) {
            const uint64_t j = i - seg_off;
            if (j == 0) v = novel_to - novel_from;
            else if (novel_from + j - 1 < novel_to) v = novel[novel_from + j - 1];
        }
        out[i] = v;
    }
}

// The all-reduced window: the statistics are added to global_stats (two windows may be in flight), the keys of every
// other rank are inserted without joining the novel list (they are not shipped again).  Errors are ORed into err.
__global__ void dm_k_window_import(const unsigned long long* __restrict__ in, uint32_t world, uint32_t self_rank,
                                   uint64_t seg_keys, unsigned long long* __restrict__ global_stats, DmTable t,
                                   unsigned int* err, int with_keys) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = tid; i < DM_STATS_WORDS; i += nth) atomicAdd(global_stats + i, in[i]);
    if (!with_keys) return;
    for (uint32_t r = 0; r < world; ++r) {
        if (r == self_rank) continue;            // own keys are already in the local table
        const uint64_t seg = (uint64_t)DM_STATS_WORDS + (uint64_t)r * (1ull + seg_keys);
        const uint64_t cnt = in[seg];
        for (uint64_t j = tid; j < cnt && j < seg_keys; j += nth) {
            unsigned long long k = in[seg + 1 + j];
            if (k) dm_table_insert(t, k, err, false);
        }
    }
}

// dm_import_known: keys[0, n) into the table, not joining the novel list.
__global__ void dm_k_insert_keys(DmTable t, const unsigned long long* __restrict__ keys, uint64_t n, unsigned int* err) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long k = keys[i];
        if (k) dm_table_insert(t, k, err, false);
    }
}

// ---------------------------------------------------------------------------------------------- known-set export
// dm_export_known: the table's non-zero slots compacted into a buffer (order unspecified), then an LSD radix sort of
// the compacted keys, 8 bits per pass, in place of a host copy of the whole table and a host sort.  A pass whose digit
// is the same for every key is skipped (the digit histograms of all eight passes come from one read of the keys).
// A pass: per CTA tile the count of each digit (digit-major, counts[d * n_tiles + tile]), one exclusive scan of those
// counts, which gives each (digit, tile) its first output position, then a stable scatter.
#define DMK_THREADS 256                              // = DMK_BINS: thread t owns digit t where a CTA works per digit
#define DMK_ITEMS 16
#define DMK_TILE (DMK_THREADS * DMK_ITEMS)           // keys (compaction: slots) per CTA tile
#define DMK_BINS 256
#define DMK_PASSES 8
#define DMK_HIST_WORDS (DMK_PASSES * DMK_BINS + 2)   // the digit histograms, the compacted count, the scan's total

// keys[0, n) <- the non-zero slots of slots[0, n_slots), at most cap of them; *n_out += n.  Per tile a warp ballot per
// round of loads, the warps' counts scanned in the CTA and one atomic offset per tile.
__global__ void __launch_bounds__(DMK_THREADS) dm_k_known_compact(const unsigned long long* __restrict__ slots,
                                                                  uint64_t n_slots, unsigned long long* __restrict__ keys,
                                                                  uint64_t cap, unsigned int* n_out) {
    __shared__ unsigned int s_warp[DMK_THREADS / 32];
    __shared__ unsigned int s_base;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt = dm_lanemask_lt();
    for (uint64_t tile = (uint64_t)blockIdx.x * DMK_TILE; tile < n_slots; tile += (uint64_t)gridDim.x * DMK_TILE) {
        unsigned long long v[DMK_ITEMS];
        unsigned int b[DMK_ITEMS];
        unsigned int cnt = 0;
        for (uint32_t i = 0; i < DMK_ITEMS; ++i) {
            const uint64_t j = tile + (uint64_t)i * DMK_THREADS + threadIdx.x;
            v[i] = j < n_slots ? slots[j] : 0ull;
            b[i] = __ballot_sync(0xffffffffu, v[i] != 0ull);
            cnt += __popc(b[i]);
        }
        if (lane == 0) s_warp[warp] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int tot = 0;
            for (uint32_t w = 0; w < DMK_THREADS / 32; ++w) {
                const unsigned int c = s_warp[w];
                s_warp[w] = tot;
                tot += c;
            }
            s_base = tot ? atomicAdd(n_out, tot) : 0u;
        }
        __syncthreads();
        uint64_t pos = (uint64_t)s_base + s_warp[warp];
        for (uint32_t i = 0; i < DMK_ITEMS; ++i) {
            if (v[i]) {
                const uint64_t p = pos + __popc(b[i] & lt);
                if (p < cap) keys[p] = v[i];
            }
            pos += __popc(b[i]);
        }
        __syncthreads();                                 // s_warp and s_base are the next tile's
    }
}

// hist[p * 256 + d] += the keys of keys[0, n) whose digit p (bits 8p .. 8p+7) is d, for all eight digits.
__global__ void __launch_bounds__(DMK_THREADS) dm_k_known_digits(const unsigned long long* __restrict__ keys, uint64_t n,
                                                                 unsigned int* __restrict__ hist) {
    __shared__ unsigned int s_h[DMK_PASSES * DMK_BINS];
    for (uint32_t i = threadIdx.x; i < DMK_PASSES * DMK_BINS; i += DMK_THREADS) s_h[i] = 0;
    __syncthreads();
    for (uint64_t j = (uint64_t)blockIdx.x * DMK_THREADS + threadIdx.x; j < n; j += (uint64_t)gridDim.x * DMK_THREADS) {
        const unsigned long long k = keys[j];
        for (uint32_t p = 0; p < DMK_PASSES; ++p) atomicAdd(&s_h[p * DMK_BINS + (uint32_t)((k >> (8 * p)) & 0xFF)], 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < DMK_PASSES * DMK_BINS; i += DMK_THREADS)
        if (s_h[i]) atomicAdd(hist + i, s_h[i]);
}

// One CTA per tile of keys[0, n): counts[d * gridDim.x + blockIdx.x] = the tile's keys whose digit at `shift` is d.
__global__ void __launch_bounds__(DMK_THREADS) dm_k_known_count(const unsigned long long* __restrict__ keys, uint64_t n,
                                                                uint32_t shift, unsigned int* __restrict__ counts) {
    __shared__ unsigned int s_h[DMK_BINS];
    s_h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * DMK_TILE + threadIdx.x;
    for (uint32_t i = 0; i < DMK_ITEMS; ++i) {
        const uint64_t j = base + (uint64_t)i * DMK_THREADS;
        if (j < n) atomicAdd(&s_h[(uint32_t)((keys[j] >> shift) & 0xFF)], 1u);
    }
    __syncthreads();
    counts[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x] = s_h[threadIdx.x];
}

// One CTA per tile: out[offsets[d * gridDim.x + blockIdx.x] + r] = the tile's r-th key (in input order) whose digit at
// `shift` is d (offsets: the exclusive scan of dm_k_known_count's counts).  Round i takes keys tile + i * 256 + t: per
// warp the lanes of equal digit are found with eight ballots, per digit the warps are ranked in lane order, so the
// scatter is stable.
__global__ void __launch_bounds__(DMK_THREADS) dm_k_known_scatter(const unsigned long long* __restrict__ in, uint64_t n,
                                                                  uint32_t shift, const unsigned int* __restrict__ offsets,
                                                                  unsigned long long* __restrict__ out) {
    __shared__ unsigned int s_cnt[DMK_THREADS / 32][DMK_BINS];   // per warp and digit: the round's keys, then their offset
    __shared__ unsigned int s_run[DMK_BINS];                     // per digit: where the tile's next key goes
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt = dm_lanemask_lt();
    s_run[threadIdx.x] = offsets[(uint64_t)threadIdx.x * gridDim.x + blockIdx.x];
    const uint64_t base = (uint64_t)blockIdx.x * DMK_TILE + threadIdx.x;
    for (uint32_t i = 0; i < DMK_ITEMS; ++i) {
        const uint64_t j = base + (uint64_t)i * DMK_THREADS;
        const bool valid = j < n;
        const unsigned long long k = valid ? in[j] : 0ull;
        const uint32_t d = (uint32_t)((k >> shift) & 0xFF);
        unsigned int peers = __ballot_sync(0xffffffffu, valid);
        for (uint32_t bit = 0; bit < 8; ++bit) {
            const unsigned int m = __ballot_sync(0xffffffffu, (d >> bit) & 1u);
            peers &= ((d >> bit) & 1u) ? m : ~m;
        }
        for (uint32_t x = lane; x < DMK_BINS; x += 32) s_cnt[warp][x] = 0;
        __syncwarp();
        const unsigned int rank = __popc(peers & lt);
        if (valid && rank == 0) s_cnt[warp][d] = __popc(peers);
        __syncthreads();
        unsigned int run = s_run[threadIdx.x];           // thread t: digit t over the warps
        for (uint32_t w = 0; w < DMK_THREADS / 32; ++w) {
            const unsigned int c = s_cnt[w][threadIdx.x];
            s_cnt[w][threadIdx.x] = run;
            run += c;
        }
        s_run[threadIdx.x] = run;
        __syncthreads();
        if (valid) out[s_cnt[warp][d] + rank] = k;
        __syncthreads();                                 // s_cnt is the next round's
    }
}

// The export's scratch, carved from one block: two key buffers of kcap keys (the compaction's output and the sort's
// ping-pong), the per-tile digit counts of a pass, the scan's tile sums and DMK_HIST_WORDS words of histograms.  Returns
// its bytes (base may be nullptr).
struct DmKnownScratch {
    unsigned long long* a;
    unsigned long long* b;
    unsigned int* counts;                            // DMK_BINS * dm_known_tiles(kcap)
    unsigned int* tile_sums;
    unsigned int* hist;                              // [8 * 256] histograms, [2048] compacted keys, [2049] scan total
    uint64_t kcap;
};

static inline uint64_t dm_known_tiles(uint64_t n) { return (n + DMK_TILE - 1) / DMK_TILE; }

static inline uint64_t dm_known_scratch(void* base, uint64_t kcap, DmKnownScratch* s) {
    const uint64_t n_counts = (uint64_t)DMK_BINS * (dm_known_tiles(kcap) > 0 ? dm_known_tiles(kcap) : 1);
    const uint64_t keys = 2 * kcap * 8, counts = 4 * n_counts, sums = 4 * (dm_alert_tiles(n_counts) + 1);
    if (base && s) {
        uint8_t* p = (uint8_t*)base;
        s->a = (unsigned long long*)p;
        s->b = (unsigned long long*)(p + kcap * 8);
        s->counts = (unsigned int*)(p + keys);
        s->tile_sums = (unsigned int*)(p + keys + counts);
        s->hist = (unsigned int*)(p + keys + counts + sums);
        s->kcap = kcap;
    }
    return keys + counts + sums + 4 * DMK_HIST_WORDS;
}

// The passes the sort runs for n keys with the digit histograms hist: the bit shifts of the digits not shared by every
// key, lowest first, into shifts[]; their number.
static inline uint32_t dm_known_passes(const unsigned int* hist, uint64_t n, uint32_t* shifts) {
    uint32_t np = 0;
    for (uint32_t p = 0; p < DMK_PASSES; ++p) {
        bool constant = false;
        for (uint32_t d = 0; d < DMK_BINS; ++d) constant |= hist[p * DMK_BINS + d] == n;
        if (!constant) shifts[np++] = 8 * p;
    }
    return np;
}
