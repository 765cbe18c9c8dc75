// dm_kernels_window.cuh -- the multi-GPU window exchange (dm_window_export / dm_window_import) and the known-set
// import (dm_import_known).
//
// Buffer layout (uint64 words): [0, DM_STATS_WORDS) the statistics delta, summed over ranks; with keys, then per rank r
// a segment [count, key_0 .. key_{seg_keys-1}] that only rank r fills, so the SUM all-reduce concatenates the
// segments.  libdmdetect passes seg_keys = DM_WINDOW_KEYS; the host side of an export is dm_window_keys (dm_host.h).
#pragma once
#include "dm_device.cuh"

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
