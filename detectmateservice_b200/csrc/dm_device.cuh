// dm_device.cuh -- device-side data structures and helpers shared by the kernels.
//
// Compiles with nvcc for sm_90a (the product) and, with -DDM_EMU, with g++ against
// tests/emu/cuda_emu.h (CPU emulation used only by the test tier).
#pragma once
#ifdef DM_EMU
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/dmdetect.h"
#include "dm_hash.h"

#define DM_STATS_WORDS (8 + DM_MAX_KEYS)   // layout of dm_stats_t as uint64 words

// Monitored keys, as the kernels see them (copied to shared memory per CTA).
struct DmKeys {
    uint32_t n;
    uint32_t len[DM_MAX_KEYS];
    uint64_t salt[DM_MAX_KEYS];
    uint8_t bytes[DM_MAX_KEYS][DM_MAX_KEYLEN];
    // fused-kernel key identification.  With w_c = bytes q-4..q-1 and w_b = bytes q-8..q-5 in
    // front of an '=' at q (later byte in the higher bits), key k matches its last
    // min(len,8) bytes iff ((w_c ^ tailbits) & tailmask) | ((w_b ^ midbits) & midmask) == 0.
    // The field-start delimiter (byte q-len-1) sits in word dsel (0 = w_c, 1 = w_b, 2 = w_a =
    // bytes q-12..q-9) at bit offset dshift, for keys shorter than 12 bytes.
    uint32_t tailbits[DM_MAX_KEYS];
    uint32_t tailmask[DM_MAX_KEYS];
    uint32_t midbits[DM_MAX_KEYS];
    uint32_t midmask[DM_MAX_KEYS];
    uint32_t dsel[DM_MAX_KEYS];
    uint32_t dshift[DM_MAX_KEYS];
    // the same patterns packed for one 16-byte shared-memory load per key, in the order the
    // fused kernel tries the keys: longest first, so that a key that is a suffix of another
    // ("res" / "xres") is only considered when the longer one does not match.
    uint32_t order[DM_MAX_KEYS];
    alignas(16) uint32_t pat[DM_MAX_KEYS][4];      // [slot] = {tailbits, tailmask, midbits, midmask} of key order[slot]
};

static inline void dm_keys_finalize_host(DmKeys* k) {
    for (uint32_t i = 0; i < k->n; ++i) {
        const uint32_t len = k->len[i];
        uint32_t tb = 0, tm = 0, mb = 0, mm = 0;
        for (uint32_t d = 1; d <= len && d <= 8; ++d) {            // d = distance from the '='
            const uint32_t byte = k->bytes[i][len - d];
            if (d <= 4) { tb |= byte << (8 * (4 - d)); tm |= 0xFFu << (8 * (4 - d)); }
            else { mb |= byte << (8 * (8 - d)); mm |= 0xFFu << (8 * (8 - d)); }
        }
        k->tailbits[i] = tb; k->tailmask[i] = tm; k->midbits[i] = mb; k->midmask[i] = mm;
        const uint32_t dd = len + 1;                                // distance of the delimiter
        k->dsel[i] = dd <= 12 ? (dd - 1) / 4 : 3;                   // 3 = not in the 12-byte window
        k->dshift[i] = dd <= 12 ? 8 * (4 * ((dd - 1) / 4 + 1) - dd) : 0;
    }
    for (uint32_t i = 0; i < k->n; ++i) k->order[i] = i;
    for (uint32_t i = 1; i < k->n; ++i) {                           // insertion sort, longest first, stable
        const uint32_t v = k->order[i];
        uint32_t j = i;
        while (j > 0 && k->len[k->order[j - 1]] < k->len[v]) { k->order[j] = k->order[j - 1]; --j; }
        k->order[j] = v;
    }
    for (uint32_t s = 0; s < k->n; ++s) {
        const uint32_t i = k->order[s];
        k->pat[s][0] = k->tailbits[i]; k->pat[s][1] = k->tailmask[i];
        k->pat[s][2] = k->midbits[i]; k->pat[s][3] = k->midmask[i];
    }
}

// Per-batch header written by the kernels, read back by the host.
struct DmBatchHeader {
    unsigned long long n_newlines;
    unsigned long long n_lines;        // records in the batch (R-tok L1)
    unsigned long long n_anomalies;    // records with score > 0
    unsigned int anomaly_list_count;   // entries appended to the anomaly list (may exceed cap)
    unsigned int error;                // DM_DEVERR_* bits
};

#define DM_DEVERR_TABLE_FULL 1u
#define DM_DEVERR_TOO_MANY_LINES 2u
#define DM_DEVERR_NOVEL_OVERFLOW 4u

// Known-set table: open addressing, linear probing, 0 = empty slot.
struct DmTable {
    unsigned long long* slots;
    uint32_t mask;                     // capacity - 1
    uint32_t limit;                    // max entries (load limit)
    unsigned long long* count;         // entries
    unsigned long long* novel;         // keys inserted since creation, in insertion order
    unsigned long long* novel_count;
    uint32_t novel_cap;
};

__device__ __forceinline__ uint32_t dm_slot_of(uint64_t key, uint32_t mask) {
    return ((uint32_t)key ^ (uint32_t)(key >> 32)) & mask;
}

// Read-only probe (detection launches: the table does not change while they run).
__device__ __forceinline__ bool dm_table_contains(const DmTable& t, uint64_t key) {
    uint32_t i = dm_slot_of(key, t.mask);
    for (uint32_t probes = 0; probes <= t.mask; ++probes) {
        unsigned long long v = __ldg(t.slots + i);
        if (v == key) return true;
        if (v == 0ull) return false;
        i = (i + 1) & t.mask;
    }
    return false;
}

// Probe that tolerates concurrent inserts (training launches).
__device__ __forceinline__ bool dm_table_contains_volatile(const DmTable& t, uint64_t key) {
    uint32_t i = dm_slot_of(key, t.mask);
    for (uint32_t probes = 0; probes <= t.mask; ++probes) {
        unsigned long long v = *((volatile unsigned long long*)(t.slots + i));
        if (v == key) return true;
        if (v == 0ull) return false;
        i = (i + 1) & t.mask;
    }
    return false;
}

// Returns true if this call inserted the key (it was not present).  learnt = the key was learnt from this rank's own
// records: it is appended to the novel list, which the window exchange ships to the other ranks (keys that arrive
// from peers or from dm_import_known are not shipped again).
__device__ __forceinline__ bool dm_table_insert(const DmTable& t, uint64_t key, unsigned int* err, bool learnt = true) {
    uint32_t i = dm_slot_of(key, t.mask);
    for (uint32_t probes = 0; probes <= t.mask; ++probes) {
        unsigned long long v = atomicCAS(t.slots + i, 0ull, (unsigned long long)key);
        if (v == 0ull) {
            unsigned long long c = atomicAdd(t.count, 1ull);
            if (c + 1 > t.limit) atomicOr(err, DM_DEVERR_TABLE_FULL);
            if (learnt) {
                unsigned long long j = atomicAdd(t.novel_count, 1ull);
                if (j < t.novel_cap) t.novel[j] = key; else atomicOr(err, DM_DEVERR_NOVEL_OVERFLOW);
            }
            return true;
        }
        if (v == key) return false;
        i = (i + 1) & t.mask;
    }
    atomicOr(err, DM_DEVERR_TABLE_FULL);
    return false;
}

#ifndef DM_EMU
// 4-bit mask of the bytes of w equal to the replicated byte pattern pat (bit j = byte j).
__device__ __forceinline__ uint32_t dm_nib_eq(uint32_t w, uint32_t pat) {
    uint32_t m = __vcmpeq4(w, pat) & 0x08040201u;
    return (m * 0x01010101u) >> 24;
}

// 16-bit mask over a 16-byte chunk.
__device__ __forceinline__ uint32_t dm_mask16_eq(uint4 v, uint32_t pat) {
    return dm_nib_eq(v.x, pat) | (dm_nib_eq(v.y, pat) << 4) | (dm_nib_eq(v.z, pat) << 8) |
           (dm_nib_eq(v.w, pat) << 12);
}
#endif

__device__ __forceinline__ uint32_t dm_lanemask_lt() {
#ifdef DM_EMU
    return (1u << (threadIdx.x & 31)) - 1u;
#else
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
#endif
}

// Named barriers (PTX bar.sync / bar.arrive; counts are in threads).
__device__ __forceinline__ void dm_bar_sync(int id, int count) {
#ifdef DM_EMU
    emu_bar_sync(id, (unsigned)count);
#else
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
#endif
}
__device__ __forceinline__ void dm_bar_arrive(int id, int count) {
#ifdef DM_EMU
    emu_bar_arrive(id, (unsigned)count);
#else
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
#endif
}

// Arguments of the warp-per-record kernels (dm_kernels_v1.cuh, dm_kernels_format.cuh).
struct DmKeys;
struct DmDetectArgs {
    const uint8_t* buf;
    const uint32_t* line_start;
    const DmBatchHeader* hdr_in;      // n_lines
    DmBatchHeader* hdr;
    const DmKeys* keys;
    DmTable table;
    uint8_t* flags;
    float* scores;
    uint64_t out_cap;
    dm_anomaly_t* anomalies;
    uint32_t anomaly_cap;
    unsigned long long* stats;
    uint64_t line_lo, line_hi;        // records [line_lo, min(line_hi, n_lines)) are processed
    uint64_t nbytes;                  // message size
    const void* combos;               // lanes / format kernel with combinations: const DmMonitors* (else NULL)
};

// The thread-per-record kernels' arguments for a message K_A has indexed into line_start (line_lo / line_hi are set
// per launch).
static inline DmDetectArgs dm_detect_args(const uint8_t* buf, uint64_t nbytes, const uint32_t* line_start, DmBatchHeader* hdr,
                                          const DmKeys* keys, DmTable table, uint8_t* flags, float* scores, uint64_t out_cap,
                                          dm_anomaly_t* anomalies, uint32_t anomaly_cap, unsigned long long* stats,
                                          const void* combos) {
    DmDetectArgs a{};
    a.buf = buf; a.nbytes = nbytes; a.line_start = line_start; a.hdr_in = hdr; a.hdr = hdr; a.keys = keys; a.table = table;
    a.flags = flags; a.scores = scores; a.out_cap = out_cap; a.anomalies = anomalies; a.anomaly_cap = anomaly_cap;
    a.stats = stats; a.combos = combos;
    return a;
}

// The grid of a grid-stride kernel over n items, `threads` per CTA: one item per thread, capped at max_grid CTAs, at
// least one CTA.
static inline unsigned dm_grid(uint64_t n, unsigned threads, uint64_t max_grid) {
    const uint64_t want = (n + threads - 1) / threads;
    const uint64_t grid = want < max_grid ? want : max_grid;
    return (unsigned)(grid > 1 ? grid : 1);
}

// Their grid.  The number of records is only known on the device: the grid is sized for the most the message can hold
// (one per byte pair, at most max_lines), capped at max_grid CTAs (the kernels stride); CTAs past the last record leave
// after one compare.
static inline unsigned dm_detect_grid(uint64_t nbytes, uint64_t max_lines, unsigned threads, uint64_t max_grid) {
    return dm_grid(nbytes / 2 + 1 < max_lines ? nbytes / 2 + 1 : max_lines, threads, max_grid);
}

// ---------------------------------------------------------------------------------------
// byte-level helpers shared by the kernels (R-tok, DESIGN.md section 2)
// ---------------------------------------------------------------------------------------
// look-back states of the row index kernel (dm_kernels_index.cuh)
#define DMT_ST_AGG 1ull
#define DMT_ST_PREFIX 2ull

// 0x80 in every byte of w that equals the byte replicated in pat (pat bytes < 0x80).
__device__ __forceinline__ uint32_t dm_eqflags(uint32_t w, uint32_t pat) {
    const uint32_t x = w ^ pat;
    const uint32_t a = (x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
    return ~(a | x) & 0x80808080u;
}
// 0x80 flags (bits 7,15,23,31) -> 4-bit mask
__device__ __forceinline__ uint32_t dm_flags_to_nib(uint32_t f) { return (f * 0x00204081u) >> 28; }

__device__ __forceinline__ uint32_t dm_ld8(const uint8_t* __restrict__ buf, uint64_t p) { return __ldg(buf + p); }
__device__ __forceinline__ uint32_t dm_ld32(const uint8_t* __restrict__ buf, uint64_t p_aligned) {
    return __ldg(reinterpret_cast<const uint32_t*>(buf + p_aligned));
}

// Byte-wise check that key k ends right before the '=' at q and starts at a field start
// (R-tok L4 delimiter; quote parity is re-checked later, see file header).  The last
// `skip_tail` key bytes are known to match already.
__device__ __forceinline__ bool dm_key_check(const uint8_t* __restrict__ buf, uint64_t q, uint32_t k, const DmKeys& sk,
                                             uint32_t skip_tail) {
    const uint32_t len = sk.len[k];
    if (q < len) return false;
    const uint64_t st = q - len;
    if (st > 0) {
        const uint32_t c = dm_ld8(buf, st - 1);
        if (c != 0x20u && c != 0x27u && c != 0x0Au) return false;
    }
    const uint32_t n = len - skip_tail;
    for (uint32_t i = 0; i < n; ++i)
        if (dm_ld8(buf, st + i) != sk.bytes[k][i]) return false;
    return true;
}

// Which monitored key (if any) ends right before the '=' at q?  Word-parallel: the 12 bytes
// in front of q are compared against every key's precomputed patterns.
__device__ __forceinline__ int dm_key_identify(const uint8_t* __restrict__ buf, uint64_t q, const DmKeys& sk) {
    if (q < 12) {
        for (uint32_t k = 0; k < sk.n; ++k)
            if (dm_key_check(buf, q, k, sk, 0)) return (int)k;
        return -1;
    }
    const uint64_t a0 = (q - 12) & ~3ull;
    const uint32_t sh = (uint32_t)((q - 12) & 3) * 8;
    const uint32_t x0 = dm_ld32(buf, a0), x1 = dm_ld32(buf, a0 + 4), x2 = dm_ld32(buf, a0 + 8), x3 = dm_ld32(buf, a0 + 12);
    const uint32_t w_a = __funnelshift_r(x0, x1, sh);    // bytes q-12 .. q-9
    const uint32_t w_b = __funnelshift_r(x1, x2, sh);    // bytes q-8 .. q-5
    const uint32_t w_c = __funnelshift_r(x2, x3, sh);    // bytes q-4 .. q-1
    // first (= longest) key whose last min(len,8) bytes stand in front of the '='
    uint32_t slot = 0xFFFFFFFFu;
    for (uint32_t s = 0; s < sk.n; ++s) {
        const uint4 p = *reinterpret_cast<const uint4*>(sk.pat[s]);
        const uint32_t diff = ((w_c ^ p.x) & p.y) | ((w_b ^ p.z) & p.w);
        if (diff == 0 && slot == 0xFFFFFFFFu) slot = s;
    }
    if (slot == 0xFFFFFFFFu) return -1;
    const uint32_t k = sk.order[slot];
    const uint32_t len = sk.len[k];
    if (len <= 8) {
        // field-start delimiter (R-tok L4); a shorter key that is a suffix of this one cannot
        // be a field start here either, its delimiter position holds a byte of this key
        const uint32_t sel = sk.dsel[k];
        const uint32_t dw = sel == 0 ? w_c : (sel == 1 ? w_b : w_a);
        const uint32_t d = (dw >> sk.dshift[k]) & 0xFFu;
        return (d == 0x20u || d == 0x27u || d == 0x0Au) ? (int)k : -1;
    }
    // keys longer than the 8 compared bytes: finish byte by byte, then fall back to the others
    if (dm_key_check(buf, q, k, sk, 8)) return (int)k;
    for (uint32_t s = slot + 1; s < sk.n; ++s) {
        const uint32_t k2 = sk.order[s];
        if (dm_key_check(buf, q, k2, sk, 0)) return (int)k2;
    }
    return -1;
}

// dm_fp64 of the value that starts at vpos: ends at the first space outside double quotes
// (parity counted from the value start, R-tok L5), at '\n', or at the end of the message.
// Works on 16-byte blocks; quote parity is carried with shift/xor prefix tricks, no branches
// on the data inside a block.
__device__ __forceinline__ uint64_t dm_hash_value(const uint8_t* __restrict__ buf, uint64_t nbytes, uint64_t vpos) {
    DmHashState st;
    dm_hash_init(st);
    uint32_t n = 0, in_q = 0;                 // in_q: 0 or 0x80808080
    uint64_t a = vpos & ~3ull;
    const uint32_t sh = (uint32_t)(vpos & 3) * 8;
    uint32_t lo = (a < nbytes) ? dm_ld32(buf, a) : 0u;
    uint64_t pos = vpos;
    for (;;) {
        const uint32_t x1 = (a + 4 < nbytes) ? dm_ld32(buf, a + 4) : 0u;
        const uint32_t x2 = (a + 8 < nbytes) ? dm_ld32(buf, a + 8) : 0u;
        const uint32_t x3 = (a + 12 < nbytes) ? dm_ld32(buf, a + 12) : 0u;
        const uint32_t x4 = (a + 16 < nbytes) ? dm_ld32(buf, a + 16) : 0u;
        uint32_t w[4];
        w[0] = __funnelshift_r(lo, x1, sh); w[1] = __funnelshift_r(x1, x2, sh);
        w[2] = __funnelshift_r(x2, x3, sh); w[3] = __funnelshift_r(x3, x4, sh);
        lo = x4;
        a += 16;
        uint32_t nvtot = 16;
        uint32_t q_state = in_q;
        uint32_t term[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t nl = dm_eqflags(w[i], 0x0A0A0A0Au);
            const uint32_t sp = dm_eqflags(w[i], 0x20202020u);
            const uint32_t dq = dm_eqflags(w[i], 0x22222222u);
            uint32_t incl = dq ^ (dq << 8);
            incl ^= incl << 16;                                     // quote parity up to and including each byte
            const uint32_t before = (incl << 8) ^ q_state;          // in-quote state in front of each byte
            term[i] = nl | (sp & ~before);
            q_state ^= (uint32_t)((int32_t)incl >> 31) & 0x80808080u;   // parity of the whole word
        }
#pragma unroll
        for (int i = 3; i >= 0; --i)
            if (term[i]) nvtot = 4u * i + ((uint32_t)(__ffs(term[i]) - 1) >> 3);
        const uint64_t rem = nbytes > pos ? nbytes - pos : 0;
        if (rem < nvtot) nvtot = (uint32_t)rem;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (nvtot > 4u * i) {
                const uint32_t nb = nvtot - 4u * i;                 // valid bytes of this word (>= 1)
                dm_hash_word(st, nb >= 4u ? w[i] : (w[i] & ((1u << (8 * nb)) - 1u)));
            }
        }
        n += nvtot;
        if (nvtot < 16) break;
        in_q = q_state;
        pos += 16;
    }
    return dm_hash_final(st, n);
}

// 16-bit mask of the bytes of a 16-byte chunk equal to the byte replicated in pat
__device__ __forceinline__ uint32_t dm_chunk_mask(const uint4& v, uint32_t pat) {
    return dm_flags_to_nib(dm_eqflags(v.x, pat)) | (dm_flags_to_nib(dm_eqflags(v.y, pat)) << 4) |
           (dm_flags_to_nib(dm_eqflags(v.z, pat)) << 8) | (dm_flags_to_nib(dm_eqflags(v.w, pat)) << 12);
}

