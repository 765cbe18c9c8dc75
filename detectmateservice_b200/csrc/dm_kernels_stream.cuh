// dm_kernels_stream.cuh -- the "stream" variant of the fused tokenizer + detector (sm_90a), default.
//
// Replaces, per record: MatcherParser field extraction + NewValueDetector.train / .detect of the
// un-vendored detectmatelibrary, which the reference drives one record at a time from
// Service.process (/root/reference/src/service/core.py:201-203).  Rules: DESIGN.md R-tok L1-L7 and
// R-spec 1-4.  ONE kernel per message in steady state (261 B per 256-byte record, read once):
//
//   * every warp owns a CONTIGUOUS range of 1 KiB rows and streams it through a private shared-memory
//     ring of four slots: one elected lane issues TMA bulk copies (cp.async.bulk global -> shared,
//     mbarrier complete_tx) one row ahead; no LDG in the row loop, no registers held by loads in
//     flight, and every later access to the text (key bytes in front of an '=', the value behind
//     it) is a shared-memory read at any alignment;
//   * row phase (32 bytes per lane): count '\n' (for the record index, see epilogue), flag the '='
//     bytes with SIMD-in-register compares into one byte-ordered 32-bit mask per lane, rank every '='
//     of the row across the warp (a prefix of the lanes' counts: rank order = message order), and
//     look them up by rank, 32 per step, so that the row's '=' are spread evenly over the lanes (the
//     ranks go through a small per-warp array in shared memory, 128 per round): the 4 bytes in front
//     of the '=' index a perfect-hash table of the monitored keys' last four bytes (3-byte keys:
//     delimiter + key).  Only hits -- about as many as there are monitored fields, a quarter of the
//     '=' -- go to the per-warp field queue, in rank order (one ballot per step);
//   * field phase (one queued field per lane, 32 at a time): finish the key compare (bytes 5..12
//     in front of the '=' and the field-start delimiter), find the value's end from ONE byte
//     class ("stop bytes" < 0x23: space, '"', '\n', controls) over a 32-byte window, dm_fp64,
//     table probe;
//   * quote parity (R-tok L2-L4) and first-occurrence-wins (L6) are NOT tracked on that path: they
//     can only change the outcome for a value that is not in the table, so exactly those
//     candidates are re-checked exactly: by their own lane, walking the record backwards
//     (dmx_verify_thread), or -- second instantiation, for streams in which candidates are
//     frequent -- a whole batch at a time from what lies between consecutive queue entries
//     (dmx_verify_chain);
//   * the record index of a byte is needed for ALERTS only: alerts are staged as (offset of the
//     record's first byte, field) and the last CTA to finish runs the epilogue -- prefix of the
//     per-CTA '\n' counts, batch header, record index of each alert, atomics on scores / flags /
//     statistics, anomaly list.  The zero-fill of flags / scores is spread over all CTAs.
//
// CTAs are small (2 warps): a CTA's slot is free again as soon as its two warps are through, and
// consecutive launches overlap (programmatic dependent launch): a launch never waits for its
// predecessor kernel; what has to be ordered is ordered by sequence numbers in device memory
// (DmxShared): scratch buffers rotate over DMX_NPAR sets and a launch starts only after the
// epilogue of the launch DMX_NPAR before it has finished; epilogues run one after the other.
#pragma once
#include "dm_kernels_index.cuh"    // dm_pdl_*, dm_launch_pdl_smem; byte helpers in dm_device.cuh

#define DMX_ROW 1024u
#define DMX_ROW_LOG2 10
#define DMX_SLOTS 4u
#define DMX_PRE 16u                         // every slot also holds the 16 bytes in front of its row (key bytes of its first
#define DMX_POST 64u                        // '=') and the 64 bytes behind it (value of its last field): a field only ever
#define DMX_SLOT (DMX_PRE + DMX_ROW + DMX_POST)   // touches its own slot
#define DMX_RING (DMX_SLOT * DMX_SLOTS)     // bytes of ring per warp
#ifndef DMX_WARPS
#define DMX_WARPS 2
#endif
#define DMX_THREADS (DMX_WARPS * 32)
#define DMX_ROUND 128u                      // '=' of a row looked up per round (4 per lane)
#define DMX_QCAP 256u                       // field queue entries per warp (circular; a round adds at most 128 to at most 31)
#define DMX_DEPTH 1u                        // rows loaded ahead (queued fields may then be up to 3 rows old)
#define DMX_L1 512u                         // most slots of the level-1 key table
#define DMX_WIN 32u                         // bytes of value looked at by the fast path
#define DMX_FULL 0x40u                      // level-1 info: the four bytes decide alone (3-byte key + delimiter)
#define DMX_RING_SMEM (DMX_WARPS * DMX_RING)
#ifndef DMX_MIN_CTAS
#define DMX_MIN_CTAS 16                     // CTAs per SM the register allocation aims at
#endif
#define DMB_ROW 512u                        // row of the boundary kernels (dm_k_rowcount / dm_k_bound)

#define DM_DEVERR_ANOMALY_OVERFLOW 8u

struct DmxL1 { uint32_t pat; uint32_t info; };      // info (7 bits): 0 = empty, else (first key of the chain + 1) | DMX_FULL

// Monitored keys as the stream kernel sees them.
struct DmxKeyTab {
    uint32_t n;
    uint32_t mult;                           // level-1 slot of the 4 bytes t in front of an '=': (t * mult) >> shift
    uint32_t shift;
    uint32_t l1_slots;
    uint32_t n_short;                        // keys of 1..2 bytes: tried one by one after a level-1 miss
    uint32_t short_idx[DM_MAX_KEYS];
    uint32_t len[DM_MAX_KEYS];
    uint32_t next[DM_MAX_KEYS];              // next key (index + 1) with the same last four bytes, 0 = none
    uint64_t salt[DM_MAX_KEYS];
    alignas(16) uint32_t pat[DM_MAX_KEYS][4];   // {bits, mask} of bytes q-8..q-5 and {bits, mask} of bytes q-12..q-9
    DmxL1 l1[DMX_L1];                        // (the first l1_slots are used; everything up to there is copied to shared memory)
    uint8_t bytes[DM_MAX_KEYS][DM_MAX_KEYLEN];  // read from global memory (slow paths only)
};
#define DMX_KEYTAB_HOT(slots) (offsetof(DmxKeyTab, l1) + (size_t)(slots) * sizeof(DmxL1))

// Ordering state of one handle (device memory, zeroed at creation).
#define DMX_NPAR 4u                          // launches in flight: scratch buffers rotate over this many sets
struct DmxShared {
    unsigned int done_ctr[2 * DMX_NPAR];     // CTAs of launch (seq % 8) that have finished their rows
    unsigned long long epi_done_seq;         // sequence number of the last launch whose epilogue is complete
    unsigned long long zero_bound[DMX_NPAR]; // [seq % NPAR]: records of detect message seq-NPAR: launch seq's CTAs zero-fill
                                             // that many output entries between them, its epilogue does the rest (if any)
    unsigned int slow_batches[DMX_NPAR];     // [seq % NPAR]: field-phase batches of launch seq that held a candidate
    unsigned int error;                      // DM_DEVERR_* bits of every launch with error_acc set since the host last
                                             // read and cleared them (dm_sync): a later header no longer hides them
};

struct DmxArgs {
    const uint8_t* buf;
    uint64_t nbytes;
    uint32_t n_rows;
    uint32_t rows_per_warp;
    const DmxKeyTab* keys;
    DmTable table;
    uint32_t rows_per_cta;
    uint32_t ring_smem;                      // bytes of dynamic shared memory in front of the key table
    unsigned short* row_cnt;                 // '\n' per row (this launch's parity)
    unsigned int* cta_cnt;                   // '\n' per CTA (this launch's parity)
    uint32_t ctas_per_grp;                   // CTAs per thread of the epilogue's prefix
    dm_anomaly_t* alerts;                    // staged alerts of this launch: {line = '\n' between the start of the 512-byte
                                             // row and the record start, mask = field, offset = record start}
    unsigned int* alert_count;
    uint32_t alert_cap;
    uint8_t* flags;
    float* scores;
    uint64_t out_cap;
    dm_anomaly_t* anomalies;
    uint32_t anomaly_cap;
    DmBatchHeader* hdr;
    unsigned long long* stats;
    uint64_t n_train_lines;
    uint64_t max_lines;
    DmxShared* sh;
    unsigned long long seq;                  // 1, 2, 3 ... per handle
    const unsigned long long* bound_ptr;     // message with training AND detection records: byte offset of the
                                             // first detection record (dm_k_bound), else NULL
    uint32_t keep_error;                     // the epilogue ORs into hdr->error instead of assigning it
    unsigned int* error_acc;                 // the detect epilogue also ORs the header's final error bits into this word
                                             // (&sh->error), or NULL
    unsigned long long* timeline;            // diagnostics (DM_STREAM_TIMELINE=1): per CTA {smid, t_start, t_rows_done, t_exit},
                                             // then 8 epilogue stamps (globaltimer ns); else NULL
    uint32_t keytab_bytes;                   // bytes of the key table that go to shared memory (multiple of 16)
    unsigned long long* hint;                // (host-mapped) written by the detect epilogue: (batches with a candidate << 32) | rows
};

__device__ __forceinline__ unsigned long long dmx_now() {
#ifndef DM_EMU
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
#else
    return 0;
#endif
}

// ---------------------------------------------------------------------------------------
// host: key tables
// ---------------------------------------------------------------------------------------
// Returns false if no perfect hash was found (<= 96 patterns in 512 slots: a few thousand multipliers at worst).
static inline bool dmx_keytab_build(const DmKeys& k, DmxKeyTab* t) {
    memset(t, 0, sizeof(*t));
    t->n = k.n;
    uint32_t pats[3 * DM_MAX_KEYS], info[3 * DM_MAX_KEYS], np = 0;
    static const uint8_t delims[3] = {0x20, 0x27, 0x0A};
    for (uint32_t i = 0; i < k.n; ++i) {
        const uint32_t L = k.len[i];
        t->len[i] = L;
        t->salt[i] = k.salt[i];
        memcpy(t->bytes[i], k.bytes[i], DM_MAX_KEYLEN);
        uint32_t mb = 0, mm = 0, ab = 0, am = 0;
        for (uint32_t d = 5; d <= L && d <= 12; ++d) {              // d = distance from the '='
            const uint32_t byte = k.bytes[i][L - d];
            if (d <= 8) { mb |= byte << (8 * (8 - d)); mm |= 0xFFu << (8 * (8 - d)); }
            else { ab |= byte << (8 * (12 - d)); am |= 0xFFu << (8 * (12 - d)); }
        }
        t->pat[i][0] = mb; t->pat[i][1] = mm; t->pat[i][2] = ab; t->pat[i][3] = am;
        if (L <= 2) { t->short_idx[t->n_short++] = i; continue; }
        if (L == 3) {
            for (int d = 0; d < 3; ++d) {
                pats[np] = (uint32_t)delims[d] | ((uint32_t)k.bytes[i][0] << 8) | ((uint32_t)k.bytes[i][1] << 16) | ((uint32_t)k.bytes[i][2] << 24);
                info[np++] = (i + 1) | DMX_FULL;
            }
            continue;
        }
        const uint32_t p = (uint32_t)k.bytes[i][L - 4] | ((uint32_t)k.bytes[i][L - 3] << 8) | ((uint32_t)k.bytes[i][L - 2] << 16) |
                           ((uint32_t)k.bytes[i][L - 1] << 24);
        uint32_t j = 0;
        for (; j < np; ++j)
            if (pats[j] == p) break;
        if (j < np) {                                               // same last four bytes as an earlier key: chain
            uint32_t c = (info[j] & 0x3Fu) - 1;
            while (t->next[c]) c = t->next[c] - 1;
            t->next[c] = i + 1;
        } else {
            pats[np] = p; info[np++] = i + 1;
        }
    }
    for (uint32_t lg = 6; lg <= 9; ++lg) {
        const uint32_t slots = 1u << lg;
        if (np > slots / 4 && lg < 9) continue;
        uint64_t x = 0x9E3779B97F4A7C15ull;
        for (int trial = 0; trial < 2000000; ++trial) {
            x = dm_splitmix64(x);
            const uint32_t mult = (uint32_t)x | 1u;
            bool used[DMX_L1];
            memset(used, 0, sizeof(used));
            bool ok = true;
            for (uint32_t j = 0; j < np && ok; ++j) {
                const uint32_t s = (pats[j] * mult) >> (32 - lg);
                if (used[s]) ok = false;
                used[s] = true;
            }
            if (!ok) continue;
            t->mult = mult; t->shift = 32 - lg; t->l1_slots = slots;
            for (uint32_t s = 0; s < slots; ++s) {                  // an empty slot holds a pattern that hashes elsewhere
                uint32_t p = 0;
                while (((p * mult) >> (32 - lg)) == s) ++p;
                t->l1[s].pat = p; t->l1[s].info = 0;
            }
            for (uint32_t j = 0; j < np; ++j) {
                const uint32_t s = (pats[j] * mult) >> (32 - lg);
                t->l1[s].pat = pats[j]; t->l1[s].info = info[j];
            }
            return true;
        }
    }
    return false;
}

// ---------------------------------------------------------------------------------------
// device: shared-memory ring fed by TMA bulk copies
// ---------------------------------------------------------------------------------------
#ifndef DM_EMU
__device__ __forceinline__ uint32_t dmx_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void dmx_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void dmx_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void dmx_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void dmx_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ unsigned long long dmx_ld_acquire(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void dmx_st_release(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t dmx_ldcg32(const uint32_t* p) { return __ldcg(p); }
#else
static inline unsigned long long dmx_ld_acquire(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline uint32_t dmx_ldcg32(const uint32_t* p) { return *p; }
static inline void dmx_st_release(unsigned long long* p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
#endif

// One warp's ring: issue() is called by lane 0 only, wait() by the whole warp.  Row r lives in slot r % SLOTS as
// [16 bytes in front of it | the row | 64 bytes behind it].
struct DmxRing {
    uint8_t* ring;                  // DMX_RING bytes
    const uint8_t* buf;
    uint64_t nb16;                  // readable extent of the message (nbytes rounded up to 16)
    uint32_t r0;                    // first row of this warp
#ifndef DM_EMU
    uint32_t ring_s, bar_s;
#endif

    __device__ __forceinline__ void issue(uint32_t i) const {
        const uint32_t row = r0 + i;
        const uint32_t slot = row & (DMX_SLOTS - 1);
        const uint32_t pre = row ? DMX_PRE : 0u;           // (the 16 bytes in front of the message are filled in by hand)
        const uint64_t off = (uint64_t)row * DMX_ROW - pre;
        const uint64_t left = nb16 - off;
        const uint32_t bytes = left < DMX_SLOT - DMX_PRE + pre ? (uint32_t)left : DMX_SLOT - DMX_PRE + pre;
#ifndef DM_EMU
        const uint32_t bar = bar_s + 8u * slot;
        dmx_mbar_expect_tx(bar, bytes);
        dmx_bulk_g2s(ring_s + slot * DMX_SLOT + DMX_PRE - pre, buf + off, bytes, bar);
#else
        memcpy(ring + slot * DMX_SLOT + DMX_PRE - pre, buf + off, bytes);
#endif
    }
    __device__ __forceinline__ void wait(uint32_t i) const {
#ifndef DM_EMU
        dmx_mbar_wait(bar_s + 8u * ((r0 + i) & (DMX_SLOTS - 1)), (i / DMX_SLOTS) & 1u);
#else
        (void)i;
        __syncwarp();
#endif
    }
};

__device__ __forceinline__ uint32_t dmx_ld32(const uint8_t* ring, uint32_t ring_off) { return *reinterpret_cast<const uint32_t*>(ring + ring_off); }

__device__ __forceinline__ bool dmx_is_delim(uint32_t d) { return d == 0x20u || d == 0x27u || d == 0x0Au; }

// 0x80 in every byte of w that is below 0x23 (space, '!', '"', '\n', controls)
__device__ __forceinline__ uint32_t dmx_stopflags(uint32_t w) {
    const uint32_t t = (w | 0x80808080u) - 0x23232323u;
    return ~(t | w) & 0x80808080u;
}

// Which monitored key (if any) ends right before the '=' at q, given the level-1 hit `info`?  Reads
// bytes q-12 .. q-5 from the field's ring slot (the 16 bytes in front of the message are '\n').
__device__ __forceinline__ int dmx_resolve_key(const uint8_t* ring, uint32_t ra, const uint8_t* __restrict__ buf, uint32_t q, uint32_t info,
                                               const DmxKeyTab& sk, const DmxKeyTab* gk) {
    if (info & DMX_FULL) return (int)(info & 0x3Fu) - 1;
    const uint32_t base = (ra - 12u) & ~3u;              // ra = place of the '=' in the ring (q = its offset in the message)
    const uint32_t sh = (ra & 3u) * 8u;
    const uint32_t x0 = dmx_ld32(ring, base), x1 = dmx_ld32(ring, base + 4), x2 = dmx_ld32(ring, base + 8);
    const uint32_t w_a = __funnelshift_r(x0, x1, sh);     // bytes q-12 .. q-9
    const uint32_t w_b = __funnelshift_r(x1, x2, sh);     // bytes q-8 .. q-5
    for (uint32_t k1 = info & 0x3Fu; k1; k1 = sk.next[k1 - 1]) {
        const uint32_t k = k1 - 1;
        const uint4 p = *reinterpret_cast<const uint4*>(sk.pat[k]);
        if ((((w_b ^ p.x) & p.y) | ((w_a ^ p.z) & p.w)) != 0) continue;
        const uint32_t L = sk.len[k];
        if (L <= 11u) {                                   // the field-start delimiter (R-tok L4) is inside the window
            const uint32_t d = L <= 7u ? (w_b >> (8u * (7u - L))) & 0xFFu : (w_a >> (8u * (11u - L))) & 0xFFu;
            if (dmx_is_delim(d)) return (int)k;
            continue;
        }
        // keys of 12 bytes and more: the rest byte by byte from global memory
        if (q < L) continue;
        const uint32_t st = q - L;
        bool ok = st == 0 || dmx_is_delim(dm_ld8(buf, st - 1));
        for (uint32_t i = 0; ok && i + 12u < L; ++i) ok = dm_ld8(buf, st + i) == gk->bytes[k][i];
        if (ok) return (int)k;
    }
    return -1;
}

// Keys of one or two bytes (none in the usual configurations): t = the 4 bytes in front of the '='.
__device__ __forceinline__ uint32_t dmx_short_key(uint32_t t, const DmxKeyTab& sk, const DmxKeyTab* gk) {
    for (uint32_t s = 0; s < sk.n_short; ++s) {
        const uint32_t k = sk.short_idx[s];
        if (sk.len[k] == 2u) {
            if ((t >> 16) == ((uint32_t)gk->bytes[k][0] | ((uint32_t)gk->bytes[k][1] << 8)) && dmx_is_delim((t >> 8) & 0xFFu))
                return (k + 1) | DMX_FULL;
        } else if ((t >> 24) == (uint32_t)gk->bytes[k][0] && dmx_is_delim((t >> 16) & 0xFFu)) {
            return (k + 1) | DMX_FULL;
        }
    }
    return 0;
}

// Value length by the letter of R-tok L3/L5 (slow path: values longer than the window).
__device__ __forceinline__ uint32_t dmx_value_len_slow(const uint8_t* __restrict__ buf, uint64_t nbytes, uint64_t vpos) {
    uint32_t par = 0;
    uint64_t p = vpos;
    for (; p < nbytes; ++p) {
        const uint32_t c = dm_ld8(buf, p);
        if (c == 0x0Au || (c == 0x20u && !par)) break;
        if (c == 0x22u) par ^= 1u;
    }
    return (uint32_t)(p - vpos);
}

// Exact re-check of one candidate by ONE thread: is the '=' at q the first true field (R-tok L2-L6)
// with key k of its record?  Walks the record backwards in 16-byte chunks: finds its first byte,
// the quote parity of the candidate's field start, and whether an earlier field start with the same
// key and the same parity exists (keys hold no quotes, so the parity at an earlier key's start is
// the parity at its '=').  The candidate's own key bytes and delimiter are known to match.
__device__ __forceinline__ bool dmx_verify_thread(const uint8_t* __restrict__ buf, uint32_t q, uint32_t k, const DmxKeyTab* gk,
                                                  uint32_t* line_start) {
    const uint32_t L = gk->len[k];
    const uint32_t p0 = q - L;
    uint32_t par = 0, s = 0;
    bool dup = false;
    if (p0 > 0) {
        for (long long c = (long long)((p0 - 1) >> 4); c >= 0; --c) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(buf + c * 16));
            const uint32_t cb = (uint32_t)c * 16u;
            uint32_t keep = 0xFFFFu;
            if (p0 - cb < 16u) keep = (1u << (p0 - cb)) - 1u;               // bytes in front of p0 only
            const uint32_t nl = dm_chunk_mask(v, 0x0A0A0A0Au) & keep;
            bool found = false;
            if (nl) {
                const uint32_t top = 31u - (uint32_t)__clz((int)nl);
                s = cb + top + 1u;
                keep &= ~((2u << top) - 1u);                                // bytes of this record only
                found = true;
            }
            const uint32_t dq = dm_chunk_mask(v, 0x22222222u) & keep;
            uint32_t eq = dm_chunk_mask(v, 0x3D3D3D3Du) & keep;
            while (eq) {
                const uint32_t j = (uint32_t)__ffs(eq) - 1u;
                eq &= eq - 1u;
                const uint32_t e = cb + j;
                if (e < L) continue;
                const uint32_t pe = par ^ ((uint32_t)__popc(dq >> (j + 1u)) & 1u);       // quotes in (e, p0)
                if (pe) continue;
                const uint32_t ks = e - L;
                bool ok = ks == 0 || dmx_is_delim(dm_ld8(buf, ks - 1));
                for (uint32_t i = 0; ok && i < L; ++i) ok = dm_ld8(buf, ks + i) == gk->bytes[k][i];
                if (ok) dup = true;
            }
            par ^= (uint32_t)__popc(dq) & 1u;
            if (found) break;
        }
    }
    *line_start = s;
    return par == 0 && !dup;
}

// ---------------------------------------------------------------------------------------
// Chained re-check of a whole batch of queued fields (the field phase's slow path).
//
// dmx_verify_thread walks a candidate's record back to its first byte: fine when candidates are rare
// (one in a thousand records), quadratic when a long record holds dozens of them -- BASELINE config 5,
// where every `kN="v .. res=quoted x"` filler carries a quoted look-alike of a monitored key.  The
// queue already holds EVERY '=' that ends a monitored key, so what a candidate needs is only what lies
// between consecutive entries: each lane scans the bytes between its predecessor's '=' and its own
// (last '\n', parity of '"' behind it), a segmented scan over the lanes turns that into (first byte of
// the record, quote parity at the '=') per entry, and a second one ORs the keys of the true fields
// (parity 0) seen earlier in the same record -- R-tok L2, L4, L6 for all 32 entries at once.  The
// state behind the last entry is carried to the next batch (DmxCarry): a long record is walked once,
// not once per candidate.
//
// What the queue guarantees: entries are in message order, in every row (the row phase enqueues a row's
// hits in the rank order of their '=', rounds and rows one after the other).  So everything in front of a
// batch's first entry has left the queue: that is what the history (no carried state) or the carried state
// stands for, and nothing still queued lies in front of any of its entries.  Batches that hold an entry of
// a row in which a lane has more than four '=' (`dense` rows) still go to dmx_verify_thread as a whole.
// Order no longer needs that; it keeps the always-exact one-by-one re-check running inside chained
// streams, where the emulator tier compares the two on the same batches
// (tests/test_emu_tile.py::test_emu_lookalikes_and_duplicates counts them).
// ---------------------------------------------------------------------------------------
// (inlined: as a real call the function's own register demand counts against the kernel's 64 and ptxas spills in the
// row loop; inlined the rare path costs the detect kernel nothing)
#ifndef DM_NOINLINE
#define DM_NOINLINE __forceinline__
#endif
#ifdef DM_EMU
static unsigned long long g_emu_chain_stats[8];      // [0] candidates decided by the chain, [2] those of batches not chained
#endif
struct DmxCarry {
    uint32_t qh_next;        // queue index of the entry right behind the batch this state describes
    uint32_t last_q;         // the largest '=' offset of that batch
    uint32_t ls;             // first byte of the record it lies in
    uint32_t par;            // quote parity at last_q
    uint32_t seen;           // keys of the true fields of that record up to and including last_q
    int dense_row;           // last row (of this warp's) in which a lane had more than four '=' (see above)
};

// bytes [lb, q): offset behind the last '\n' (found) and the parity of '"' behind it (else of the whole interval)
__device__ __forceinline__ void dmx_scan_back(const uint8_t* __restrict__ buf, uint32_t lb, uint32_t q, bool& found, uint32_t& ls,
                                              uint32_t& par) {
    found = false; ls = lb; par = 0;
    if (q <= lb) return;
    for (long long c = (long long)((q - 1u) >> 4); c >= (long long)(lb >> 4); --c) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(buf + c * 16));
        const uint32_t cb = (uint32_t)c * 16u;
        uint32_t keep = 0xFFFFu;
        if (q - cb < 16u) keep = (1u << (q - cb)) - 1u;
        if (cb < lb) keep &= ~((1u << (lb - cb)) - 1u);
        const uint32_t nl = dm_chunk_mask(v, 0x0A0A0A0Au) & keep;
        if (nl) {
            const uint32_t top = 31u - (uint32_t)__clz((int)nl);
            ls = cb + top + 1u;
            keep &= ~((2u << top) - 1u);
            found = true;
        }
        par ^= (uint32_t)__popc(dm_chunk_mask(v, 0x22222222u) & keep) & 1u;
        if (found) break;
    }
}

// Which monitored key ends right before the '=' at e, starting at a field start of the record that begins at ls (-1: none)?
// Byte-wise from global memory: the slow paths' counterpart of dmx_resolve_key.
__device__ __forceinline__ int dmx_key_at(const uint8_t* __restrict__ buf, const DmxKeyTab* gk, uint32_t nk, uint32_t e, uint32_t ls) {
    for (uint32_t k = 0; k < nk; ++k) {
        const uint32_t L = gk->len[k];
        if (e < ls + L) continue;
        const uint32_t ks = e - L;
        bool ok = ks == ls || dmx_is_delim(dm_ld8(buf, ks - 1u));
        for (uint32_t i = L; ok && i > 0; --i) ok = dm_ld8(buf, ks + i - 1u) == gk->bytes[k][i - 1u];
        if (ok) return (int)k;
    }
    return -1;
}

// Warp-collective: the record that holds byte q0 - 1 (q0 = an '=' offset): *ls = its first byte, *par_q0 = parity of '"' in
// [ls, q0), return value = keys of its true fields (R-tok L2/L4/L5) whose '=' lies in [ls, q0).  Two passes over the
// bytes themselves, 512 per step: backwards for the last '\n' in front of q0, then forwards with the running parity.
__device__ __forceinline__ uint32_t dmx_history(const uint8_t* __restrict__ buf, const DmxKeyTab* gk, uint32_t q0, uint32_t* ls_out, uint32_t* par_q0) {
    const uint32_t lane = threadIdx.x & 31, full = 0xffffffffu;
    const uint4* b16 = reinterpret_cast<const uint4*>(buf);
    uint32_t ls = 0;
    {
        const long long ctop = (long long)((q0 - 1u) >> 4);                  // (q0 > 0: an '=' is never the first byte of a key)
        for (long long c0 = ctop; c0 >= 0; c0 -= 32) {
            const long long c = c0 - (31 - (long long)lane);
            uint32_t nl = 0;
            if (c >= 0) {
                nl = dm_chunk_mask(__ldg(b16 + c), 0x0A0A0A0Au);
                if (c == ctop && (q0 & 15u)) nl &= (1u << (q0 & 15u)) - 1u;
            }
            const uint32_t has = __ballot_sync(full, nl != 0u);
            if (has) {
                const int top = 31 - __clz((int)has);
                const uint32_t bits = __shfl_sync(full, nl, top);
                ls = (uint32_t)(c0 - (31 - top)) * 16u + (31u - (uint32_t)__clz((int)bits)) + 1u;
                break;
            }
        }
    }
    uint32_t seen = 0, run = 0;
    const uint32_t nk = gk->n;
    for (uint32_t cb0 = ls & ~15u; cb0 < q0; cb0 += 512u) {
        const uint32_t cb = cb0 + 16u * lane;
        uint32_t dq = 0, eq = 0;
        if (cb < q0) {
            const uint4 v = __ldg(b16 + (cb >> 4));
            uint32_t keep = 0xFFFFu;
            if (cb < ls) keep &= ~((1u << (ls - cb)) - 1u);
            if (q0 - cb < 16u) keep &= (1u << (q0 - cb)) - 1u;
            dq = dm_chunk_mask(v, 0x22222222u) & keep;
            eq = dm_chunk_mask(v, 0x3D3D3D3Du) & keep;
        }
        const uint32_t odd = __ballot_sync(full, (__popc(dq) & 1) != 0);
        const uint32_t par_in = run ^ ((uint32_t)__popc(odd & dm_lanemask_lt()) & 1u);
        while (eq) {
            const uint32_t j = (uint32_t)__ffs(eq) - 1u;
            eq &= eq - 1u;
            if ((par_in ^ ((uint32_t)__popc(dq & ((1u << j) - 1u)) & 1u)) != 0u) continue;     // inside double quotes
            const int k = dmx_key_at(buf, gk, nk, cb + j, ls);
            if (k >= 0) seen |= 1u << k;
        }
        run ^= (uint32_t)__popc(odd) & 1u;
        __syncwarp();
    }
    *ls_out = ls;
    *par_q0 = run;
    return __reduce_or_sync(full, seen);
}

// Warp-collective.  Lane i < n holds queue entry i of the batch: '=' at qpos_in, key k_in (-1: no monitored key ends
// there, or the record is not this pass's), cand_in = its value is not in the table.  `chainable` = no entry of a dense
// row.  Returns (ok << 32) | ls: ok = 1 for the candidates that are the first true field with their key in their record,
// ls = first byte of that record.
__device__ DM_NOINLINE unsigned long long dmx_verify_chain(const uint8_t* __restrict__ buf, const DmxKeyTab* gk, DmxCarry* cy, uint32_t qh,
                                                           uint32_t n, bool chainable, uint32_t qpos_in, int k, bool cand) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t full = 0xffffffffu;
    bool ok = false;
    uint32_t ls = 0;
    if (!chainable) {
        if (cand && k >= 0) {
            ok = dmx_verify_thread(buf, qpos_in, (uint32_t)k, gk, &ls);
#ifdef DM_EMU
            __atomic_fetch_add(&g_emu_chain_stats[2], 1ull, __ATOMIC_RELAXED);
#endif
        }
        if (lane == 0) cy->qh_next = 0xFFFFFFFFu;
        __syncwarp();
        return ((unsigned long long)(ok ? 1u : 0u) << 32) | ls;
    }
    const bool inq = lane < n;
    const uint32_t qpos = inq ? qpos_in : 0xFFFFFFFFu;
    const uint32_t q_first = __shfl_sync(full, qpos, 0);
    const bool cont = cy->qh_next == qh && cy->last_q < q_first;
    uint32_t c_q = cy->last_q, c_ls = cy->ls, c_par = cy->par, c_seen = cy->seen;
    // ---- nothing carried over: the record the batch starts in is read from its first byte up to the batch's first '='
    // (history); from there on the queue speaks ----
    if (!cont) {
        c_seen = dmx_history(buf, gk, q_first, &c_ls, &c_par);
        c_q = 0xFFFFFFFFu;
    }
    uint32_t prev = __shfl_up_sync(full, qpos, 1);
    if (lane == 0) prev = c_q;
    // ---- per entry: the bytes between the previous '=' and this one ----
    bool found = false;
    uint32_t par = 0;
    if (inq && !(lane == 0 && !cont)) dmx_scan_back(buf, prev + 1u, qpos, found, ls, par);
    __syncwarp();
    bool abs_ = inq && (found || lane == 0);                          // (ls, par) already count from the record's first byte
    if (lane == 0 && !found) { ls = c_ls; par ^= c_par; }
    // ---- segmented scan: (first byte of the record, parity at the '=') of every entry ----
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(full, (par << 1) | (abs_ ? 1u : 0u), d);
        const uint32_t yl = __shfl_up_sync(full, ls, d);
        if ((int)lane >= d && !abs_) { par ^= y >> 1; ls = yl; abs_ = (y & 1u) != 0u; }
    }
    // ---- keys of the true fields seen earlier in the same record ----
    const uint32_t ls_prev = __shfl_up_sync(full, ls, 1);
    const bool head = lane == 0 ? c_ls != ls : ls_prev != ls;                 // no earlier entry of this record in the batch / the carry
    const uint32_t bit = (inq && k >= 0 && par == 0u) ? 1u << k : 0u;
    uint32_t incl = bit | ((lane == 0 && !head) ? c_seen : 0u);
    bool hd = head;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(full, incl, d);
        const uint32_t yh = __shfl_up_sync(full, hd ? 1u : 0u, d);
        if ((int)lane >= d && !hd) { incl |= y; hd = yh != 0u; }
    }
    uint32_t before = __shfl_up_sync(full, incl, 1);
    if (lane == 0) before = head ? 0u : c_seen;
    else if (head) before = 0u;
    if (cand && k >= 0) {
        ok = par == 0u && !(before & (1u << k));
#ifdef DM_EMU
        __atomic_fetch_add(&g_emu_chain_stats[0], 1ull, __ATOMIC_RELAXED);
#endif
    }
    __syncwarp();
    // ---- what the next batch needs ----
    if (lane == n - 1u) {
        cy->qh_next = qh + n;
        cy->last_q = qpos;
        cy->ls = ls;
        cy->par = par & 1u;
        cy->seen = incl;
    }
    __syncwarp();
    return ((unsigned long long)(ok ? 1u : 0u) << 32) | ls;
}

// ---------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------
// zero-fill of output entries [lo, hi): 16-byte stores where the caller's buffers allow it
__device__ __forceinline__ void dmx_zero_outputs(uint8_t* flags, float* scores, unsigned long long lo, unsigned long long hi,
                                                 uint32_t tid, uint32_t nthreads) {
    if (hi <= lo) return;
    unsigned long long v0 = lo, v1 = lo;
    if ((((uintptr_t)flags) | ((uintptr_t)scores)) % 16 == 0) {
        v0 = (lo + 15ull) & ~15ull;
        v1 = hi & ~15ull;
        if (v1 < v0) v0 = v1 = lo;
    }
    for (unsigned long long i = v0 + (unsigned long long)tid * 16; i < v1; i += nthreads * 16ull) {
        *reinterpret_cast<uint4*>(flags + i) = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(scores + i + 4 * j) = make_uint4(0, 0, 0, 0);
    }
    for (unsigned long long i = lo + tid; i < v0; i += nthreads) { flags[i] = 0; scores[i] = 0.0f; }
    for (unsigned long long i = v1 + tid; i < hi; i += nthreads) { flags[i] = 0; scores[i] = 0.0f; }
}

// The bytes of a 16-byte chunk equal to `pat` as bits 8b+i of the result (byte b of word i), i.e. UNORDERED: cheaper
// than a mask in position order, and all that is done with it is to count or to enumerate.
__device__ __forceinline__ uint32_t dmx_chunk_bits(const uint4& v, uint32_t pat) {
    const uint32_t f0 = dm_eqflags(v.x, pat), f1 = dm_eqflags(v.y, pat), f2 = dm_eqflags(v.z, pat), f3 = dm_eqflags(v.w, pat);
    return (f0 >> 7) | (f1 >> 6) | (f2 >> 5) | (f3 >> 4);
}

// The '=' of a 16-byte chunk IN BYTE ORDER (bit i = byte i: the set bits enumerate them in message order), with the
// three-instruction zero-byte test, which is exact except that a run of '<' (0x3C = '=' ^ 1) right behind an '=' in the
// same 32-bit word is flagged as well (the borrow of the subtraction).  Harmless: the bytes in front of such a position
// hold that '=' within the last three, an '=' is part of no monitored key (dm_create rejects it) and is no field-start
// delimiter, so the key lookup of the position fails like that of any other '=' that ends no monitored key.  ('\n' is
// counted, so it keeps the exact test.)
__device__ __forceinline__ uint32_t dmx_loose_bits(const uint4& v, uint32_t pat) {
    const uint32_t x0 = v.x ^ pat, x1 = v.y ^ pat, x2 = v.z ^ pat, x3 = v.w ^ pat;
    const uint32_t f0 = (x0 - 0x01010101u) & ~x0 & 0x80808080u, f1 = (x1 - 0x01010101u) & ~x1 & 0x80808080u;
    const uint32_t f2 = (x2 - 0x01010101u) & ~x2 & 0x80808080u, f3 = (x3 - 0x01010101u) & ~x3 & 0x80808080u;
    return dm_flags_to_nib(f0) | (dm_flags_to_nib(f1) << 4) | (dm_flags_to_nib(f2) << 8) | (dm_flags_to_nib(f3) << 12);
}
__device__ __forceinline__ uint32_t dmx_eq_bits(const uint4& v) { return dmx_loose_bits(v, 0x3D3D3D3Du); }

// Inclusive prefix sum over the lanes of a warp.  (The shuffle's own "source lane exists" predicate guards each add,
// so no lane index compare is issued per step.)
__device__ __forceinline__ uint32_t dmx_warp_incl_sum(uint32_t v) {
#pragma unroll
    for (uint32_t d = 1; d < 32u; d <<= 1) {
#ifndef DM_EMU
        asm("{\n\t.reg .u32 t;\n\t.reg .pred p;\n\t"
            "shfl.sync.up.b32 t|p, %0, %1, 0, -1;\n\t"
            "@p add.u32 %0, %0, t;\n\t}"
            : "+r"(v)
            : "r"(d));
#else
        const uint32_t y = __shfl_up_sync(0xffffffffu, v, d);
        if ((threadIdx.x & 31) >= d) v += y;
#endif
    }
    return v;
}
template <bool TRAIN>
__device__ __forceinline__ void dmx_epilogue(const DmxArgs& a, unsigned long long* s_pre);

// (what the field phase needs of the kernel arguments sits in shared memory: a reference to the parameter block
// itself would force a copy of it into local memory)
struct DmxDrainCtx {
    const uint8_t* buf;
    uint64_t nbytes;
    DmTable table;
    const DmxKeyTab* gk;
    dm_anomaly_t* alerts;
    unsigned int* alert_count;
    unsigned int* err;
    uint32_t alert_cap;
};

// Field phase: n (<= 32) queued fields, one per lane.  Called from ONE place in the kernel (one copy of the code);
// the lanes are brought back together (__syncwarp) after every data-dependent stretch: without that they drift
// apart for the rest of the function and every later instruction is issued several times for a few lanes each.
template <bool TRAIN, bool CHAIN>
__device__ __forceinline__ void dmx_drain(const DmxDrainCtx& a, const DmxKeyTab& sk, const uint8_t* ring, const uint32_t* q, uint32_t qh,
                                          uint32_t n, uint32_t seg_base, uint32_t bound, DmxCarry* carry, uint32_t* s_slow) {
    const uint32_t lane = threadIdx.x & 31;
    const uint8_t* __restrict__ buf = a.buf;
    const uint64_t nbytes = a.nbytes;
    uint32_t qpos = 0, ra = 0;
    int k = -1;
    if (lane < n) {
        const uint32_t e = q[(qh + lane) & (DMX_QCAP - 1)];
        const uint32_t qrel = e >> 7;                                              // offset of the '=' in this warp's range
        qpos = seg_base + qrel;
        ra = (((seg_base >> DMX_ROW_LOG2) + (qrel >> DMX_ROW_LOG2)) & (DMX_SLOTS - 1)) * DMX_SLOT + DMX_PRE + (qrel & (DMX_ROW - 1));
        if (TRAIN ? (qpos < bound) : (qpos >= bound)) k = dmx_resolve_key(ring, ra, buf, qpos, e & 0x7Fu, sk, a.gk);
    }
    __syncwarp();
    const bool act = k >= 0;
    // ---- the value (R-tok L5): it ends at the first space outside double quotes counted from its start, at '\n',
    // or at the end of the message.  One byte class ("stop bytes" < 0x23) over a 32-byte window. ----
    const uint32_t vpos = qpos + 1u;
    const uint32_t vr = ra + 1u;                              // the value's place in the ring
    uint32_t w[8];
    uint32_t m = 0, lim = 0;
    if (act) {
        const uint32_t base = vr & ~3u;
        const uint32_t sh = (vr & 3u) * 8u;
        uint32_t lo = dmx_ld32(ring, base);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t hi = dmx_ld32(ring, base + 4u * (i + 1));
            w[i] = __funnelshift_r(lo, hi, sh);
            lo = hi;
        }
        const uint64_t avail = nbytes > vpos ? nbytes - vpos : 0;
        lim = avail < DMX_WIN ? (uint32_t)avail : DMX_WIN;
#pragma unroll
        for (int i = 0; i < 8; ++i) m |= dm_flags_to_nib(dmx_stopflags(w[i])) << (4 * i);
        if (lim < DMX_WIN) m &= (1u << lim) - 1u;
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) w[i] = 0;
    }
    uint32_t nv = 0xFFFFFFFFu;
    {
        uint32_t par = 0;
        while (m) {
            const uint32_t j = (uint32_t)__ffs(m) - 1u;
            m &= m - 1u;
            const uint32_t c = ring[vr + j];
            if (c == 0x0Au || (c == 0x20u && !par)) { nv = j; break; }
            if (c == 0x22u) par ^= 1u;
        }
    }
    __syncwarp();
    bool slow = false;
    if (act && nv == 0xFFFFFFFFu) {
        if (lim < DMX_WIN) nv = lim;                      // the message ends inside the window: that ends the value
        else slow = true;                                 // longer than the window
    }
    if (!act || slow) nv = 0;
    DmHashState st;
    dm_hash_init(st);
    {
        const uint32_t nmax = __reduce_max_sync(0xffffffffu, nv);     // words no lane needs are skipped by the whole warp
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (nmax <= 4u * i) break;
            if (nv > 4u * i) {
                const uint32_t nb = nv - 4u * i;
                dm_hash_word(st, nb >= 4u ? w[i] : (w[i] & ((1u << (8u * nb)) - 1u)));
            }
        }
    }
    uint64_t fp = dm_hash_final(st, nv);
    if (__any_sync(0xffffffffu, slow)) {
        if (slow) {                                       // by the letter, from global memory
            const uint32_t len = dmx_value_len_slow(buf, nbytes, vpos);
            fp = dm_fp64_bytes(buf + vpos, len);
        }
        __syncwarp();
    }
    bool cand = false;
    uint64_t ckey = 0;
    if (act) {
        ckey = dm_make_key(fp, sk.salt[k]);
        cand = !(TRAIN ? dm_table_contains_volatile(a.table, ckey) : dm_table_contains(a.table, ckey));
    }
    if (__any_sync(0xffffffffu, cand)) {
        // (how often this happens decides which instantiation the host launches next: see dmx_launch)
        if (lane == 0) s_slow[threadIdx.x >> 5] += 1u;
        uint32_t ls = 0;
        bool ok = false;
        if (CHAIN) {
            const bool chainable = !__any_sync(0xffffffffu, lane < n && (int)((qpos - seg_base) >> DMX_ROW_LOG2) <= carry->dense_row);
            const unsigned long long vr_ = dmx_verify_chain(buf, a.gk, carry, qh, n, chainable, qpos, k, cand);
            ls = (uint32_t)vr_;
            ok = (vr_ >> 32) != 0ull;
        } else {
            ok = cand && dmx_verify_thread(buf, qpos, (uint32_t)k, a.gk, &ls);      // every candidate walks its own record back
        }
        if (cand) {
            if (ok) {
                if (TRAIN) {
                    dm_table_insert(a.table, ckey, a.err);
                } else {
                    // an alert: unknown value in monitored field k of the record that starts at ls
                    uint32_t inrow = 0;
                    const uint4* b16 = reinterpret_cast<const uint4*>(buf);
                    for (uint32_t c = (ls & ~(DMX_ROW - 1)) >> 4; c < (ls >> 4); ++c)
                        inrow += (uint32_t)__popc(dm_chunk_mask(__ldg(b16 + c), 0x0A0A0A0Au));
                    if (ls & 15u)
                        inrow += (uint32_t)__popc(dm_chunk_mask(__ldg(b16 + (ls >> 4)), 0x0A0A0A0Au) & ((1u << (ls & 15u)) - 1u));
                    const unsigned int idx = atomicAdd(a.alert_count, 1u);
                    if (idx < a.alert_cap) {
                        dm_anomaly_t r;
                        r.line = inrow; r.mask = (uint32_t)k; r.offset = ls;
                        a.alerts[idx] = r;
                    }
                }
            }
        }
        __syncwarp();
    }
}

// CHAIN: candidates are re-checked batch-wise (dmx_verify_chain) instead of one by one.  Same results; the chained code
// costs the row loop about 5 % more instructions (its register demand makes ptxas rematerialise loop state), so it is a
// separate instantiation that the host picks for streams in which candidates are frequent (dmx_launch).
template <bool TRAIN, bool CHAIN>
__global__ void __launch_bounds__(DMX_THREADS, DMX_MIN_CTAS) dm_k_stream(DmxArgs a) {
#ifdef DM_EMU
    uint8_t* s_dyn = g_emu_dyn_smem.data();
#else
    extern __shared__ __align__(128) uint8_t s_dyn[];
#endif
    // dynamic shared memory: DMX_WARPS rings, then the key table up to its last level-1 slot
    const DmxKeyTab& sk = *reinterpret_cast<const DmxKeyTab*>(s_dyn + a.ring_smem);
    __shared__ uint32_t s_q[DMX_WARPS][DMX_QCAP];
    __shared__ uint16_t s_eq[DMX_WARPS][DMX_ROUND];
    __shared__ unsigned long long s_bar[DMX_WARPS][DMX_SLOTS];
    __shared__ uint32_t s_cnt[DMX_WARPS];
    __shared__ unsigned long long s_bound;
    __shared__ int s_last;
    __shared__ DmxDrainCtx s_ctx;
    __shared__ DmxCarry s_carry[DMX_WARPS];
    __shared__ uint32_t s_slow[DMX_WARPS];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt = dm_lanemask_lt();
    dm_pdl_launch_dependents();                       // the next launch may be scheduled as soon as there is room
    if (threadIdx.x == 0) {
        s_ctx.buf = a.buf; s_ctx.nbytes = a.nbytes; s_ctx.table = a.table; s_ctx.gk = a.keys; s_ctx.alerts = a.alerts;
        s_ctx.alert_count = a.alert_count; s_ctx.err = &a.hdr->error; s_ctx.alert_cap = a.alert_cap;
        if (a.timeline) {
            uint32_t smid = 0;
#ifndef DM_EMU
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
#endif
            a.timeline[4ull * blockIdx.x] = smid;
            a.timeline[4ull * blockIdx.x + 1] = dmx_now();
        }
    }
#ifdef DMX_KEYTAB_LOOP
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(a.keys);
        uint32_t* dst = reinterpret_cast<uint32_t*>(s_dyn + a.ring_smem);
        for (uint32_t i = threadIdx.x; i < a.keytab_bytes / 4u; i += DMX_THREADS) dst[i] = __ldg(src + i);
    }
#else
    // the key table comes in with ONE bulk copy issued by thread 0 (waited for right before the rows)
    __shared__ unsigned long long s_kbar;
    if (threadIdx.x == 0) {
        dmx_mbar_init(dmx_smem_u32(&s_kbar), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        dmx_mbar_expect_tx(dmx_smem_u32(&s_kbar), a.keytab_bytes);
        dmx_bulk_g2s(dmx_smem_u32(s_dyn + a.ring_smem), a.keys, a.keytab_bytes, dmx_smem_u32(&s_kbar));
    }
#endif
    if (lane == 0) {
        s_cnt[warp] = 0;
        s_slow[warp] = 0;
        if (CHAIN) { s_carry[warp].qh_next = 0xFFFFFFFFu; s_carry[warp].dense_row = -1; }
#ifndef DM_EMU
        for (uint32_t s = 0; s < DMX_SLOTS; ++s) dmx_mbar_init(dmx_smem_u32(&s_bar[warp][s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
    }
    // this launch's scratch (row counts, staged alerts) was last used by launch seq-NPAR: its epilogue must be through
    if (threadIdx.x == 0) {
        while (dmx_ld_acquire(&a.sh->epi_done_seq) + DMX_NPAR < a.seq) __nanosleep(64);
        const unsigned long long zb = *((volatile unsigned long long*)&a.sh->zero_bound[a.seq % DMX_NPAR]);
        s_bound = zb < a.out_cap ? zb : a.out_cap;
    }
    __syncthreads();
#ifndef DMX_KEYTAB_LOOP
    dmx_mbar_wait(dmx_smem_u32(&s_kbar), 0u);
#endif

    const uint64_t nbytes = a.nbytes;
    const uint32_t bound = a.bound_ptr ? (uint32_t)(*a.bound_ptr > 0xFFFFFFFFull ? 0xFFFFFFFFull : *a.bound_ptr) : (TRAIN ? 0xFFFFFFFFu : 0u);
    const uint32_t l1_mult = sk.mult, l1_shift = sk.shift, n_short = sk.n_short;
    const uint32_t gw = blockIdx.x * DMX_WARPS + warp;
    const uint64_t r0l = (uint64_t)gw * a.rows_per_warp;
    if (r0l < a.n_rows) {
        DmxRing rg;
        rg.ring = s_dyn + warp * DMX_RING;
        rg.buf = a.buf;
        rg.nb16 = (nbytes + 15ull) & ~15ull;
        rg.r0 = (uint32_t)r0l;
#ifndef DM_EMU
        rg.ring_s = dmx_smem_u32(rg.ring);
        rg.bar_s = dmx_smem_u32(&s_bar[warp][0]);
#endif
        const uint8_t* ring = rg.ring;
        const uint32_t n_own = (uint32_t)(r0l + a.rows_per_warp < a.n_rows ? a.rows_per_warp : a.n_rows - r0l);
        const uint32_t seg_base = rg.r0 * DMX_ROW;            // (messages are shorter than 4 GiB)
        const uint32_t tail_bytes = (uint32_t)(nbytes & (DMX_ROW - 1));   // valid bytes of a partial last row (0 = full)
        const uint32_t tail_row = tail_bytes ? a.n_rows - 1 : 0xFFFFFFFFu;
        uint32_t* q = s_q[warp];                               // fields waiting for the field phase: (offset in this warp's range << 7) | level-1 info
        uint16_t* eq = s_eq[warp];                             // the '=' of a lookup round by rank: offset in the row
        uint32_t qh = 0, qn = 0, nl_w = 0;
        if (rg.r0 == 0) {
            // a message starts a record: the 16 bytes "in front of it" read as '\n'
            if (lane < 4) reinterpret_cast<uint32_t*>(rg.ring)[lane] = 0x0A0A0A0Au;
            __syncwarp();
        }
        if (lane == 0) rg.issue(0);
        // lane l owns bytes [32 l, 32 l + 32) of a row; it reads its two 16-byte chunks in an order that keeps the
        // eight lanes of a shared-memory phase on different banks
        const uint32_t c_first = (lane >> 2) & 1u;

        for (uint32_t i = 0; i < n_own; ++i) {
            const uint32_t row = rg.r0 + i;
            if (i + 1 < n_own) {
                // row i+1 goes into the slot of row i-3, whose fields have left the queue (see the end of the loop body)
                __syncwarp();
                if (lane == 0) rg.issue(i + 1);
            }
            rg.wait(i);
            const uint32_t lb = (row & (DMX_SLOTS - 1)) * DMX_SLOT + DMX_PRE + lane * 32u;      // this lane's bytes in the ring
            uint4 va = *reinterpret_cast<const uint4*>(ring + lb + 16u * c_first);
            uint4 vb = *reinterpret_cast<const uint4*>(ring + lb + 16u * (1u - c_first));
            if (row == tail_row) {
                // partial last row: bytes behind the message are nobody's
                uint32_t* wa = reinterpret_cast<uint32_t*>(&va);
                uint32_t* wb = reinterpret_cast<uint32_t*>(&vb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t oa = lane * 32u + 16u * c_first + 4u * j, ob = lane * 32u + 16u * (1u - c_first) + 4u * j;
                    const uint32_t na = tail_bytes > oa ? tail_bytes - oa : 0u, nb = tail_bytes > ob ? tail_bytes - ob : 0u;
                    if (na < 4u) wa[j] = na ? (wa[j] & ((1u << (8u * na)) - 1u)) : 0u;
                    if (nb < 4u) wb[j] = nb ? (wb[j] & ((1u << (8u * nb)) - 1u)) : 0u;
                }
            }
            {
                // '\n' of the row (the epilogue turns the counts into record indices)
                const uint32_t c = (uint32_t)__popc(dmx_chunk_bits(va, 0x0A0A0A0Au)) + (uint32_t)__popc(dmx_chunk_bits(vb, 0x0A0A0A0Au));
                const uint32_t tot = __reduce_add_sync(0xffffffffu, c);
                if (lane == 0) a.row_cnt[row] = (unsigned short)tot;
                nl_w += tot;
            }
            // the '=' of this lane's 32 bytes: bit i = byte i
            uint32_t g = (dmx_eq_bits(va) << (16u * c_first)) | (dmx_eq_bits(vb) << (16u * (1u - c_first)));
            const uint32_t cnt = (uint32_t)__popc(g);
            const bool last = i + 1 == n_own;
            if (CHAIN) {
                if (__any_sync(0xffffffffu, cnt > 4u)) {            // (see dmx_verify_chain)
                    if (lane == 0) s_carry[warp].dense_row = (int)i;
                    __syncwarp();
                }
            }
            // rank of this lane's first '=' among the row's (message order): exclusive prefix of the lanes' counts
            uint32_t rank = dmx_warp_incl_sum(cnt);
            const uint32_t n_eq = __shfl_sync(0xffffffffu, rank, 31);
            rank -= cnt;
            const uint32_t rb = (row & (DMX_SLOTS - 1)) * DMX_SLOT + DMX_PRE;          // the row in the ring
            uint32_t r_lo = 0;                                                        // first rank of the round
            bool row_done;
            do {
                // ---- ranks [r_lo, r_lo + DMX_ROUND): offsets in the row -> s_eq[rank - r_lo].  Lane j then looks up
                // ranks j, j + 32, ... of the round: the 4 bytes in front of the '=' (shared memory, any alignment)
                // -> perfect-hash table; the hits go to the field queue in rank order, i.e. in message order ----
                {
                    while (g && rank < r_lo + DMX_ROUND) {
                        eq[rank - r_lo] = (uint16_t)(lane * 32u + (uint32_t)__ffs(g) - 1u);
                        g &= g - 1u;
                        ++rank;
                    }
                    __syncwarp();
                    const uint32_t nr = n_eq - r_lo < DMX_ROUND ? n_eq - r_lo : DMX_ROUND;
#pragma unroll
                    for (uint32_t s = 0; s < DMX_ROUND / 32u; ++s) {
                        if (32u * s >= nr) break;
                        uint32_t off = 0, info = 0;
                        if (32u * s + lane < nr) {
                            off = eq[32u * s + lane];
                            const uint32_t at = rb + off - 4u;
                            const uint32_t t = __funnelshift_r(dmx_ld32(ring, at & ~3u), dmx_ld32(ring, (at & ~3u) + 4u), (at & 3u) * 8u);
                            const DmxL1 l = sk.l1[(t * l1_mult) >> l1_shift];
                            info = l.pat == t ? l.info : 0u;
                            if (!info && n_short) info = dmx_short_key(t, sk, a.keys);
                        }
                        const uint32_t hit = __ballot_sync(0xffffffffu, info != 0u);
                        if (info) q[(qh + qn + (uint32_t)__popc(hit & lt)) & (DMX_QCAP - 1)] = ((i * DMX_ROW + off) << 7) | info;
                        qn += (uint32_t)__popc(hit);
                    }
                    r_lo += DMX_ROUND;
                    row_done = r_lo >= n_eq;
                    __syncwarp();
                }
                // ---- full passes; at the end of a row also whatever is left of rows up to (i + 2 - SLOTS): the next
                // iteration loads row i+2 into that row's slot ----
                for (;;) {
                    uint32_t n = 0;
                    if (qn >= 32u) n = 32u;
                    else if (row_done && qn && (last || (q[qh & (DMX_QCAP - 1)] >> (7 + DMX_ROW_LOG2)) + (DMX_SLOTS - 2u) <= i)) n = qn;
                    if (!n) break;
                    dmx_drain<TRAIN, CHAIN>(s_ctx, sk, ring, q, qh, n, seg_base, bound, &s_carry[warp], s_slow);
                    qh += n;
                    qn -= n;
                }
            } while (!row_done);
        }
        if (lane == 0) {
            s_cnt[warp] = nl_w;
            if (s_slow[warp]) atomicAdd(&a.sh->slow_batches[a.seq % DMX_NPAR], s_slow[warp]);
        }
    }

    // ---- end of the CTA's rows ----
    __syncthreads();
    if (!TRAIN) {
        if (threadIdx.x == 0) {
            if (a.timeline) a.timeline[4ull * blockIdx.x + 2] = dmx_now();
            uint32_t c = 0;
            for (uint32_t w = 0; w < DMX_WARPS; ++w) c += s_cnt[w];
            a.cta_cnt[blockIdx.x] = c;
        }
        // every CTA zero-fills its share of as many output entries as message seq-2 had records.  (The previous call's
        // epilogue may still be adding ITS alerts to the same buffers: this launch's epilogue takes them out again.)
        const unsigned long long zb = s_bound;
        const unsigned long long per = (((zb + gridDim.x - 1) / gridDim.x) + 15ull) & ~15ull;
        const unsigned long long lo = per * blockIdx.x < zb ? per * blockIdx.x : zb;
        dmx_zero_outputs(a.flags, a.scores, lo, lo + per < zb ? lo + per : zb, threadIdx.x, DMX_THREADS);
        __syncthreads();
    } else if (a.timeline && threadIdx.x == 0) {
        a.timeline[4ull * blockIdx.x + 2] = dmx_now();
    }
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(&a.sh->done_ctr[a.seq % (2 * DMX_NPAR)], 1u);
        s_last = old == gridDim.x - 1 ? 1 : 0;
        if (a.timeline && !s_last) a.timeline[4ull * blockIdx.x + 3] = dmx_now();
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    dmx_epilogue<TRAIN>(a, reinterpret_cast<unsigned long long*>(s_dyn));
}

// Sum of the 8 counters of one 16-byte vector of row counts
__device__ __forceinline__ uint32_t dmx_sum8(const uint4& v) {
    return (v.x & 0xFFFFu) + (v.x >> 16) + (v.y & 0xFFFFu) + (v.y >> 16) + (v.z & 0xFFFFu) + (v.z >> 16) + (v.w & 0xFFFFu) + (v.w >> 16);
}
// '\n' counts of rows [lo, hi): vector loads that bypass L1 (other CTAs wrote them)
__device__ __forceinline__ unsigned long long dmx_count_rows(const unsigned short* cnt, uint32_t lo, uint32_t hi) {
    unsigned long long s = 0;
    uint32_t r = lo;
    for (; r < hi && (r & 7u); ++r) s += *((volatile const unsigned short*)(cnt + r));
#ifndef DM_EMU
    for (; r + 32 <= hi; r += 32) {
        const uint4 v0 = __ldcg(reinterpret_cast<const uint4*>(cnt + r)), v1 = __ldcg(reinterpret_cast<const uint4*>(cnt + r + 8));
        const uint4 v2 = __ldcg(reinterpret_cast<const uint4*>(cnt + r + 16)), v3 = __ldcg(reinterpret_cast<const uint4*>(cnt + r + 24));
        s += dmx_sum8(v0) + dmx_sum8(v1) + dmx_sum8(v2) + dmx_sum8(v3);
    }
    for (; r + 8 <= hi; r += 8) s += dmx_sum8(__ldcg(reinterpret_cast<const uint4*>(cnt + r)));
#endif
    for (; r < hi; ++r) s += *((volatile const unsigned short*)(cnt + r));
    return s;
}

// Epilogue (the last CTA of a launch): batch header, rest of the zero-fill, record index of every staged alert,
// scores / flags / statistics / anomaly list.  s_pre: DMX_THREADS + 16 words of shared memory.
template <bool TRAIN>
__device__ __forceinline__ void dmx_epilogue(const DmxArgs& a, unsigned long long* s_pre) {
    const uint32_t tid = threadIdx.x;
    unsigned long long* tl = a.timeline ? a.timeline + 4ull * gridDim.x : nullptr;
    if (tl && tid == 0) tl[0] = dmx_now();
    // epilogues run in launch order (they write the caller's outputs, the header and the statistics)
    if (tid == 0)
        while (dmx_ld_acquire(&a.sh->epi_done_seq) + 1ull < a.seq) __nanosleep(64);
    __syncthreads();
    if (tl && tid == 0) tl[1] = dmx_now();
    if (!TRAIN) {
        const uint32_t G = gridDim.x;
        // the alerts of the previous call may have landed in these output buffers after this launch's CTAs zero-filled
        // them: take them out again (its anomaly list and header are still in place); a list that overflowed is no use
        const unsigned int prev_n = *((volatile unsigned int*)&a.hdr->anomaly_list_count);
        const bool prev_lost = prev_n > a.anomaly_cap;
        for (unsigned int i = tid; i < prev_n && !prev_lost; i += DMX_THREADS) {
            const uint32_t g = dmx_ldcg32(&a.anomalies[i].line);
            if (g < a.out_cap) { a.flags[g] = 0; a.scores[g] = 0.0f; }
        }
        // per-CTA '\n' counts -> shared memory (asynchronous copies, all in flight at once) -> exclusive prefix in place
        // (thread t: CTAs [t cpt, (t+1) cpt)); the warps scan their threads' sums by shuffles
        uint32_t* s_cta = reinterpret_cast<uint32_t*>(s_pre) + 256;           // G words, behind the DMX_THREADS + 16 u64 of s_pre
        const uint32_t cpt = a.ctas_per_grp;
        for (uint32_t i = tid; i < G; i += DMX_THREADS) {
#ifndef DM_EMU
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dmx_smem_u32(s_cta + i)), "l"(a.cta_cnt + i) : "memory");
#else
            s_cta[i] = a.cta_cnt[i];
#endif
        }
#ifndef DM_EMU
        asm volatile("cp.async.wait_all;" ::: "memory");
#endif
        __syncthreads();
        {
            const uint32_t lo = tid * cpt < G ? tid * cpt : G, hi = lo + cpt < G ? lo + cpt : G;
            unsigned long long c = 0;
            for (uint32_t i = lo; i < hi; ++i) c += s_cta[i];
            unsigned long long incl = c;
            const uint32_t ln = tid & 31;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, d);
                if ((int)ln >= d) incl += y;
            }
            if (ln == 31) s_pre[DMX_THREADS + 4 + (tid >> 5)] = incl;
            __syncthreads();
            unsigned long long run = incl - c;
            for (uint32_t w = 0; w < (tid >> 5); ++w) run += s_pre[DMX_THREADS + 4 + w];
            if (tid == DMX_THREADS - 1) s_pre[DMX_THREADS + 2] = run + c;          // all '\n' of the message
            for (uint32_t i = lo; i < hi; ++i) { const uint32_t ci = s_cta[i]; s_cta[i] = (uint32_t)run; run += ci; }
        }
        __syncthreads();
        if (tid == 0) {
            const unsigned long long nl = s_pre[DMX_THREADS + 2];
            const bool tail = a.nbytes > 0 && a.buf[a.nbytes - 1] != 0x0Au;
            const unsigned long long n_lines = nl + (tail ? 1ull : 0ull);
            s_pre[DMX_THREADS] = n_lines;
            s_pre[DMX_THREADS + 1] = a.sh->zero_bound[a.seq % DMX_NPAR];
            a.sh->zero_bound[a.seq % DMX_NPAR] = n_lines;
            const unsigned int staged = *((volatile unsigned int*)a.alert_count);
            unsigned int err = (n_lines > a.max_lines || n_lines > a.out_cap) ? DM_DEVERR_TOO_MANY_LINES : 0u;
            if (staged > a.alert_cap) err |= DM_DEVERR_ANOMALY_OVERFLOW;
            a.hdr->n_anomalies = 0; a.hdr->anomaly_list_count = 0;
            err = a.keep_error ? (a.hdr->error | err) : err;     // (keep_error: dm_k_bound cleared it, TRAIN inserts set bits)
            a.hdr->error = err;
            if (a.error_acc && err) atomicOr(a.error_acc, err);
            a.hdr->n_newlines = nl;
            a.hdr->n_lines = n_lines;
            const unsigned long long tr = a.n_train_lines < n_lines ? a.n_train_lines : n_lines;
            atomicAdd(a.stats + 0, n_lines);
            atomicAdd(a.stats + 1, tr);
            atomicAdd(a.stats + 2, n_lines - tr);
            atomicAdd(a.stats + 5, (unsigned long long)a.nbytes);
        }
        __syncthreads();
        if (tl && tid == 0) tl[2] = dmx_now();
        const unsigned long long n_lines = s_pre[DMX_THREADS];
        const unsigned long long n_out = n_lines < a.out_cap ? n_lines : a.out_cap;
        {
            // the CTAs zero-filled [0, bound); more records than that when the messages grow, and everything again if
            // the previous call's anomaly list is not complete
            const unsigned long long zb = s_pre[DMX_THREADS + 1] < a.out_cap ? s_pre[DMX_THREADS + 1] : a.out_cap;
            dmx_zero_outputs(a.flags, a.scores, prev_lost ? 0ull : (zb < n_out ? zb : n_out), n_out, tid, DMX_THREADS);
        }
        __threadfence_block();
        __syncthreads();
        if (tl && tid == 0) tl[3] = dmx_now();
        const unsigned int staged = *((volatile unsigned int*)a.alert_count);
        const unsigned int n_al = staged < a.alert_cap ? staged : a.alert_cap;
        for (unsigned int i0 = 0; i0 < n_al; i0 += 2 * DMX_THREADS) {
            // two alerts per thread and round: their loads overlap
            uint32_t inrow[2], k[2], s[2];
            unsigned long long g[2];
            bool on[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const unsigned int i = i0 + tid + j * DMX_THREADS;
                on[j] = i < n_al;
                inrow[j] = 0; k[j] = 0; s[j] = 0;
                if (on[j]) {
                    inrow[j] = dmx_ldcg32(&a.alerts[i].line); k[j] = dmx_ldcg32(&a.alerts[i].mask);
                    s[j] = dmx_ldcg32(reinterpret_cast<const uint32_t*>(&a.alerts[i].offset));
                }
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                // record index = '\n' in front of the record's first byte: in front of its CTA, in the CTA's rows before its row, in its row
                const uint32_t row = s[j] >> DMX_ROW_LOG2;
                const uint32_t cta = row / a.rows_per_cta;
                g[j] = 0;
                if (on[j]) g[j] = (unsigned long long)s_cta[cta] + inrow[j] + dmx_count_rows(a.row_cnt, cta * a.rows_per_cta, row);
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (!on[j]) continue;
                bool first = false;
                if (g[j] < a.out_cap) {
                    const float old = atomicAdd(a.scores + g[j], 1.0f);
                    a.flags[g[j]] = 1;
                    first = old == 0.0f;
                }
                atomicAdd(a.stats + 8 + k[j], 1ull);
                atomicAdd(a.stats + 4, 1ull);
                if (first) { atomicAdd(&a.hdr->n_anomalies, 1ull); atomicAdd(a.stats + 3, 1ull); }
                const unsigned int idx = atomicAdd(&a.hdr->anomaly_list_count, 1u);
                if (idx < a.anomaly_cap) {
                    dm_anomaly_t r;
                    r.line = (uint32_t)g[j]; r.mask = 1u << k[j]; r.offset = s[j];
                    a.anomalies[idx] = r;
                }
            }
        }
        __syncthreads();
        if (tl && tid == 0) tl[4] = dmx_now();
    }
    if (tid == 0) {
        const unsigned int sb = *((volatile unsigned int*)&a.sh->slow_batches[a.seq % DMX_NPAR]);
        a.sh->slow_batches[a.seq % DMX_NPAR] = 0;
        if (!TRAIN && a.hint) *((volatile unsigned long long*)a.hint) = ((unsigned long long)sb << 32) | a.n_rows;
        *a.alert_count = 0;
        a.sh->done_ctr[a.seq % (2 * DMX_NPAR)] = 0;
        __threadfence();
        dmx_st_release(&a.sh->epi_done_seq, a.seq);
        if (tl) tl[5] = dmx_now();
        if (a.timeline) a.timeline[4ull * blockIdx.x + 3] = dmx_now();
    }
}

// ---------------------------------------------------------------------------------------
// messages that hold training AND detection records: where does detection start?
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dm_k_rowcount(const uint8_t* __restrict__ buf, uint64_t nbytes, uint32_t n_rows,
                                                     unsigned short* __restrict__ row_cnt) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t row = w; row < n_rows; row += nw) {
        const uint64_t off = (uint64_t)row * DMB_ROW + lane * 16u;
        uint32_t m = 0;
        if (off < nbytes) m = dm_row_nl_mask(__ldg(reinterpret_cast<const uint4*>(buf + off)), off, nbytes);
        const uint32_t tot = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(m));
        if (lane == 0) row_cnt[row] = (unsigned short)tot;
    }
}

// One CTA: byte offset of record n_train (= behind the n_train-th '\n'), nbytes if the message has fewer.
__global__ void __launch_bounds__(256) dm_k_bound(const uint8_t* __restrict__ buf, uint64_t nbytes, uint32_t n_rows,
                                                  const unsigned short* __restrict__ row_cnt, uint64_t n_train,
                                                  unsigned long long* bound_out, DmBatchHeader* hdr) {
    __shared__ unsigned long long s_sum[256];
    const uint32_t tid = threadIdx.x;
    const uint32_t per = (n_rows + 255) / 256;
    const uint32_t lo = tid * per < n_rows ? tid * per : n_rows;
    const uint32_t hi = lo + per < n_rows ? lo + per : n_rows;
    unsigned long long s = 0;
    for (uint32_t r = lo; r < hi; ++r) s += row_cnt[r];
    s_sum[tid] = s;
    __syncthreads();
    if (tid == 0) {
        hdr->error = 0;
        unsigned long long bound = nbytes;
        unsigned long long run = 0;
        uint32_t t = 0;
        while (t < 256 && run + s_sum[t] < n_train) { run += s_sum[t]; ++t; }
        if (n_train == 0) bound = 0;
        else if (t < 256) {
            uint32_t r = t * per;
            while (run + row_cnt[r] < n_train) { run += row_cnt[r]; ++r; }
            uint64_t p = (uint64_t)r * DMB_ROW;
            for (;; ++p)
                if (buf[p] == 0x0Au && ++run == n_train) break;
            bound = p + 1;
        }
        *bound_out = bound;
    }
}

// Geometry of a launch over a.n_rows rows on at most max_grid CTAs: every warp gets the same number of contiguous rows.
// Sets a.rows_per_warp / rows_per_cta / ctas_per_grp; returns the grid.
static inline unsigned dmx_geometry(DmxArgs& a, uint64_t max_grid) {
    const unsigned long long warps_max = max_grid * DMX_WARPS;
    const uint32_t rpw = (uint32_t)((a.n_rows + warps_max - 1) / warps_max);
    const unsigned long long warps = (a.n_rows + rpw - 1) / rpw;
    const unsigned grid = (unsigned)((warps + DMX_WARPS - 1) / DMX_WARPS);
    a.rows_per_warp = rpw;
    a.rows_per_cta = rpw * DMX_WARPS;
    a.ctas_per_grp = (grid + DMX_THREADS - 1) / DMX_THREADS;
    return grid;
}

#ifndef DM_EMU
// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
struct DmxScratch {
    DmxKeyTab* d_keys = nullptr;
    unsigned short* d_row_cnt[DMX_NPAR] = {};
    unsigned int* d_cta_cnt[DMX_NPAR] = {};
    unsigned short* d_bound_cnt = nullptr;
    dm_anomaly_t* d_alerts[DMX_NPAR] = {};
    unsigned int* d_alert_count = nullptr;      // NPAR words
    unsigned long long* d_bound = nullptr;
    DmxShared* d_shared = nullptr;
    uint32_t alert_cap = 0;
    uint32_t dyn_smem = 0;                      // rings + key table
    uint64_t max_rows = 0;
    unsigned long long seq = 0;
    int ctas_per_sm = 0;
    int max_grid = 0;
    bool overlap = false;                       // programmatic dependent launch between consecutive detect launches
    cudaStream_t chain_stream = nullptr;        // stream of the last launch, if it was a plain detect launch (else NULL)
    unsigned long long* d_timeline = nullptr;   // DM_STREAM_TIMELINE=1
    unsigned last_grid = 0;
    // which instantiation re-checks candidates: 0 = one by one, 1 = chained, 2 = by what the last finished message looked like
    int recheck_mode = 2;
    unsigned long long* h_hint = nullptr;       // pinned, device-mapped: (batches with a candidate << 32) | rows of that message
    bool last_chained = false;
};

static inline int dmx_scratch_create(DmxScratch* s, const DmKeys& keys, uint64_t max_batch_bytes, uint32_t alert_cap, int sm_count) {
    DmxKeyTab* t = new (std::nothrow) DmxKeyTab;
    if (!t) return DM_ERR_CUDA;
    const bool ok = dmx_keytab_build(keys, t);
    s->dyn_smem = (uint32_t)(DMX_RING_SMEM + ((DMX_KEYTAB_HOT(t->l1_slots) + 15) & ~(size_t)15));
    cudaError_t e = ok ? cudaMalloc(&s->d_keys, sizeof(DmxKeyTab)) : cudaErrorUnknown;
    if (e == cudaSuccess) e = cudaMemcpy(s->d_keys, t, sizeof(DmxKeyTab), cudaMemcpyHostToDevice);
    delete t;
    if (e != cudaSuccess) return DM_ERR_CUDA;
    s->max_rows = (max_batch_bytes + DMB_ROW - 1) / DMB_ROW + 64;
    s->alert_cap = alert_cap;
    if (cudaFuncSetAttribute(dm_k_stream<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaFuncSetAttribute(dm_k_stream<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaFuncSetAttribute(dm_k_stream<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaFuncSetAttribute(dm_k_stream<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    int per_sm = 0, per_sm_c = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dm_k_stream<false, false>, DMX_THREADS, s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_c, dm_k_stream<false, true>, DMX_THREADS, s->dyn_smem) != cudaSuccess) return DM_ERR_CUDA;
    if (per_sm_c < per_sm) per_sm = per_sm_c;                // (one geometry for both instantiations)
    {
        const char* m = getenv("DM_STREAM_RECHECK");         // thread | chain | auto (default)
        if (m && !strcmp(m, "thread")) s->recheck_mode = 0;
        else if (m && !strcmp(m, "chain")) s->recheck_mode = 1;
        else if (m && strcmp(m, "auto") && *m) return DM_ERR_ARG;
        if (cudaHostAlloc((void**)&s->h_hint, sizeof(unsigned long long), cudaHostAllocMapped) != cudaSuccess) return DM_ERR_CUDA;
        *s->h_hint = 0;
    }
    if (per_sm < 1) per_sm = 1;
    const char* cap = getenv("DM_STREAM_CTAS_PER_SM");     // tuning knob
    if (cap && atoi(cap) > 0 && atoi(cap) < per_sm) per_sm = atoi(cap);
    s->ctas_per_sm = per_sm;
    s->max_grid = sm_count * per_sm;
    if (1024u + 4u * (unsigned)s->max_grid > s->dyn_smem) s->max_grid = (int)((s->dyn_smem - 1024u) / 4u);   // (epilogue: per-CTA prefix in shared memory)
    for (unsigned b = 0; b < DMX_NPAR; ++b) {
        if (cudaMalloc(&s->d_row_cnt[b], s->max_rows * sizeof(unsigned short)) != cudaSuccess) return DM_ERR_CUDA;
        if (cudaMalloc(&s->d_cta_cnt[b], (size_t)s->max_grid * sizeof(unsigned int)) != cudaSuccess) return DM_ERR_CUDA;
        if (cudaMalloc(&s->d_alerts[b], (size_t)alert_cap * sizeof(dm_anomaly_t)) != cudaSuccess) return DM_ERR_CUDA;
    }
    if (cudaMalloc(&s->d_bound_cnt, s->max_rows * sizeof(unsigned short)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMalloc(&s->d_alert_count, DMX_NPAR * sizeof(unsigned int)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMemset(s->d_alert_count, 0, DMX_NPAR * sizeof(unsigned int)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMalloc(&s->d_bound, sizeof(unsigned long long)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMalloc(&s->d_shared, sizeof(DmxShared)) != cudaSuccess) return DM_ERR_CUDA;
    if (cudaMemset(s->d_shared, 0, sizeof(DmxShared)) != cudaSuccess) return DM_ERR_CUDA;
    const char* tl = getenv("DM_STREAM_TIMELINE");
    if (tl && atoi(tl) == 1) {
        if (cudaMalloc(&s->d_timeline, ((size_t)s->max_grid * 4 + 8) * sizeof(unsigned long long)) != cudaSuccess) return DM_ERR_CUDA;
        cudaMemset(s->d_timeline, 0, ((size_t)s->max_grid * 4 + 8) * sizeof(unsigned long long));
    }
    return DM_OK;
}

static inline void dmx_scratch_destroy(DmxScratch* s) {
    cudaFree(s->d_keys);
    for (unsigned b = 0; b < DMX_NPAR; ++b) { cudaFree(s->d_row_cnt[b]); cudaFree(s->d_cta_cnt[b]); cudaFree(s->d_alerts[b]); }
    cudaFree(s->d_bound_cnt); cudaFree(s->d_alert_count); cudaFree(s->d_bound); cudaFree(s->d_shared); cudaFree(s->d_timeline);
    if (s->h_hint) cudaFreeHost(s->h_hint);
    *s = DmxScratch();
}

// Enqueue the kernels for one message.  Returns the number of kernels launched or < 0.  accumulate_errors: the message's
// error bits also go to the handle's error word (DmxShared::error), for callers whose header a later message overwrites.
static inline int dmx_launch(DmxScratch* s, const uint8_t* d_buf, uint64_t nbytes, uint64_t n_train_lines, DmTable table,
                             uint8_t* d_flags, float* d_scores, uint64_t out_cap, dm_anomaly_t* d_anoms, uint32_t anomaly_cap,
                             DmBatchHeader* d_hdr, unsigned long long* d_stats, uint64_t max_lines, cudaStream_t st,
                             bool allow_overlap, bool accumulate_errors, void (*mark)(void*, cudaStream_t, int), void* mark_ctx) {
    const uint32_t n_rows = (uint32_t)((nbytes + DMX_ROW - 1) / DMX_ROW);
    const uint32_t b_rows = (uint32_t)((nbytes + DMB_ROW - 1) / DMB_ROW);
    if (n_rows == 0) return 0;
    if (b_rows > s->max_rows) return DM_ERR_CAPACITY;
    DmxArgs a;
    a.buf = d_buf; a.nbytes = nbytes; a.n_rows = n_rows;
    a.keys = s->d_keys; a.table = table;
    a.flags = d_flags; a.scores = d_scores; a.out_cap = out_cap; a.anomalies = d_anoms; a.anomaly_cap = anomaly_cap;
    a.hdr = d_hdr; a.stats = d_stats; a.n_train_lines = n_train_lines; a.max_lines = max_lines;
    a.sh = s->d_shared; a.alert_cap = s->alert_cap; a.bound_ptr = nullptr; a.keep_error = 0; a.timeline = s->d_timeline; a.ring_smem = DMX_RING_SMEM;
    a.error_acc = accumulate_errors ? &s->d_shared->error : nullptr;
    a.keytab_bytes = s->dyn_smem - (uint32_t)DMX_RING_SMEM;
    a.hint = s->h_hint;                                      // (unified addressing: the mapped host pointer is the device pointer)
    // chained re-check when, in the last message whose epilogue has run, at least every fourth row had a batch with a
    // candidate (both instantiations give the same results; this only picks the faster one for the stream at hand)
    bool chained = s->recheck_mode == 1;
    if (s->recheck_mode == 2) {
        const unsigned long long hint = *((volatile unsigned long long*)s->h_hint);
        chained = (hint & 0xFFFFFFFFull) != 0 && (hint >> 32) * 4ull >= (hint & 0xFFFFFFFFull);
    }
    s->last_chained = chained;
    const unsigned grid = dmx_geometry(a, (uint64_t)s->max_grid);
    s->last_grid = grid;
    int launched = 0;
    auto bind = [&]() {
        a.seq = ++s->seq;
        const int p = (int)(a.seq % DMX_NPAR);
        a.row_cnt = s->d_row_cnt[p]; a.cta_cnt = s->d_cta_cnt[p]; a.alerts = s->d_alerts[p]; a.alert_count = s->d_alert_count + p;
    };
    if (n_train_lines > 0) {
        // where detection starts is only known on the device
        dm_k_rowcount<<<(unsigned)std::min<uint64_t>((b_rows + 7) / 8, 2048), 256, 0, st>>>(d_buf, nbytes, b_rows, s->d_bound_cnt);
        dm_k_bound<<<1, 256, 0, st>>>(d_buf, nbytes, b_rows, s->d_bound_cnt, n_train_lines, s->d_bound, d_hdr);
        a.bound_ptr = s->d_bound; a.keep_error = 1;
        bind();
        dm_launch_pdl_smem(chained ? dm_k_stream<true, true> : dm_k_stream<true, false>, grid, DMX_THREADS, (size_t)s->dyn_smem, st, false, a);
        launched += 3;
    }
    bind();
    const bool pdl = allow_overlap && n_train_lines == 0 && s->chain_stream == st;
    if (mark) mark(mark_ctx, st, 0);
    dm_launch_pdl_smem(chained ? dm_k_stream<false, true> : dm_k_stream<false, false>, grid, DMX_THREADS, (size_t)s->dyn_smem, st, pdl, a);
    if (mark) mark(mark_ctx, st, 1);
    s->chain_stream = st;
    ++launched;
    if (cudaGetLastError() != cudaSuccess) return DM_ERR_CUDA;
    return launched;
}
#endif  // DM_EMU
