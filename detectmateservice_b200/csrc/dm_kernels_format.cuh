// dm_kernels_format.cuh -- the MatcherParser step fused in front of the detector
// (SURVEY.md section 8a8 / 8f-3): `log_format` header extraction and `<*>` template matching on
// the device, one thread per record, feeding the same known-set table.
//
// What it replaces: detectmatelibrary.parsers.template_matcher.MatcherParser (un-vendored;
// configured at /root/reference/tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88
// and docs/getting_started.md:395-415) followed by NewValueDetector or NewValueComboDetector behind
// /root/reference/src/service/core.py:201-203.  Rules: DESIGN.md R-fmt / R-match / R-norm / R-combo.
//
//   chain     L0 C0 L1 C1 ... L(n-1) [C(n-1)]     literals L, captures C
//   match     L0 anchored at the start; every later literal at its EARLIEST occurrence at or
//             after the current position (captures are non-greedy); a chain that ends with a
//             literal anchors that literal at the END of the text; a chain that ends with a
//             capture lets it run to the end.  Equivalent to the regular expression
//             ^L0(.*?)L1(.*?)...$ with the literals escaped (checked against Python's `re`
//             in tests/test_format_matcher.py).
//   chain 0   the log_format: captures are the header variables (logFormatVariables)
//   chain 1+  the templates, matched in file order against the capture named Content;
//             the first match gives EventID (0-based template index; -1 = none) and its
//             captures are variables[0..].
#pragma once
#include "dm_device.cuh"
#include "dm_kernels_index.cuh"      // K_A, dm_pdl_wait
#include "dm_kernels_records.cuh"    // DmMonitors, dm_combo_seed / dm_combo_fold: combination monitors (dm_set_combos)

#define DM_FMT_MAX_CHAINS 64          // log_format + 63 templates
#define DM_FMT_MAX_LITS 512           // literals over all chains
#define DM_FMT_MAX_CAPTURES 32        // captures per chain: capture i is bit i of chain_need (a chain has one more literal
                                      // than captures when it ends with a literal)
#define DM_FMT_POOL_WORDS 1024        // literal text over all chains, each literal padded to 4-byte words
#define DM_FMT_MAX_LIT_LEN 255
#define DM_FMT_NONE 0xFFu
#define DM_FMT_NOT_FOUND 0xFFFFFFFFu

struct DmFormat {
    uint32_t n_chains;
    uint32_t content_capture;                         // header capture the templates apply to, DM_FMT_NONE = none
    uint32_t n_mons;
    uint32_t pad_;
    uint16_t chain_first[DM_FMT_MAX_CHAINS + 2];      // first literal of chain c (c+1: one past)
    uint8_t chain_endcap[DM_FMT_MAX_CHAINS];          // 1: the chain ends with a capture
    uint16_t lit_off[DM_FMT_MAX_LITS];                // literal i starts at pool[lit_off[i]] (word index)
    uint8_t lit_len[DM_FMT_MAX_LITS];                 // its length in bytes
    uint32_t pool[DM_FMT_POOL_WORDS];                 // little-endian words, zero padded per literal
    // monitors bound to the format: header capture index or variable index
    int32_t mon_event[DM_MAX_KEYS];
    uint8_t mon_has_event[DM_MAX_KEYS];
    uint8_t mon_source[DM_MAX_KEYS];                  // 0 = header capture, 1 = template variable
    uint8_t mon_index[DM_MAX_KEYS];                   // capture / variable index, DM_FMT_NONE = never present
    // thread-per-record kernel: captures of chain c some monitor (or the template step) reads;
    // a lane keeps only those, in slot popc(need & ((1 << capture) - 1))
    uint32_t chain_need[DM_FMT_MAX_CHAINS];
    uint32_t max_slots;                               // max over chains of popc(chain_need)
    // R-norm (MatcherParser params.remove_spaces / remove_punctuation / lowercase): the Content text
    // is rewritten without the bytes of norm_drop (a 256-bit set), letters folded, before the
    // template chains -- whose literals the host normalised the same way -- are matched against it
    uint32_t norm_flags;
    uint32_t pad2_[2];
    uint32_t norm_drop[8];
};
#ifndef DM_NORM_LOWERCASE                             // (the same bits as include/dmdetect.h)
#define DM_NORM_REMOVE_SPACES 1u
#define DM_NORM_REMOVE_PUNCTUATION 2u
#define DM_NORM_LOWERCASE 4u
#endif

// 4 text bytes starting at any byte offset (little endian).  Reads the two aligned words
// around it: up to 7 bytes past `p`, covered by the slack every message buffer carries.
// NC: the text is read-only for the whole kernel (the message) and goes through the non-coherent
// path; !NC: it is the normalised copy the SAME thread wrote earlier in this kernel (R-norm), which
// ld.global.nc must not be used on -- those loads are L2-coherent (ld.global.cg).
template <bool NC>
__device__ __forceinline__ uint32_t dm_fmt_ldw(const uint32_t* w) { return NC ? __ldg(w) : __ldcg(w); }

template <bool NC = true>
__device__ __forceinline__ uint32_t dm_fmt_load4(const uint8_t* buf, uint32_t p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(buf) + p;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    return __funnelshift_r(dm_fmt_ldw<NC>(w), dm_fmt_ldw<NC>(w + 1), (uint32_t)(a & 3u) * 8u);
}

__device__ __forceinline__ uint32_t dm_fmt_tail_mask(uint32_t nbytes) {     // nbytes in 1..4
    return 0xFFFFFFFFu >> (8u * (4u - nbytes));
}

// dm_fp64 of text[p, p+n) with word loads
template <bool NC = true>
__device__ __forceinline__ uint64_t dm_fmt_fp64(const uint8_t* buf, uint32_t p, uint32_t n) {
    DmHashState st;
    dm_hash_init(st);
    for (uint32_t i = 0; i < n; i += 4) {
        uint32_t w = dm_fmt_load4<NC>(buf, p + i);
        if (n - i < 4) w &= dm_fmt_tail_mask(n - i);
        dm_hash_word(st, w);
    }
    return dm_hash_final(st, n);
}

// =========================================================================================
// Thread-per-record variant (the decomposition of dm_kernels_lanes.cuh applied to log_format
// matching): every lane walks its own record -- sequential earliest-occurrence search with a
// sliding 8-byte window, same semantics as dm_fmt_match_chain -- keeps the captures a monitor
// reads in shared memory, then the lanes of a warp hash / probe monitor after monitor in
// lockstep.  No warp collectives; ~20x fewer warp instructions per record than one warp per
// record, at the price of 14 warps per SM on a 64k-record message.
// =========================================================================================
#define DM_FMTL_THREADS 64

// earliest q in [pos, e - len] with text[q, q+len) == literal (len >= 1), else DM_FMT_NOT_FOUND.
// Four start positions per step (one aligned word): the four compares are independent, which
// matters because a lane is one long dependent chain and only ~14 warps per SM hide latency.
template <bool NC>
__device__ __forceinline__ uint32_t dm_fmtl_find(const uint8_t* buf, uint32_t pos, uint32_t e,
                                                 const uint32_t* lit, uint32_t len) {
    if (e < pos + len) return DM_FMT_NOT_FOUND;
    const uint32_t last = e - len;
    const uint32_t w0 = lit[0];
    const uint32_t m0 = len >= 4 ? 0xFFFFFFFFu : dm_fmt_tail_mask(len);
    const uintptr_t base_addr = reinterpret_cast<uintptr_t>(buf);
    const uint32_t mis = (uint32_t)(base_addr & 3u);               // buf is word aligned in the product (mis == 0)
    uint32_t q0 = ((pos + mis) & ~3u) - mis;                       // position of the aligned word that holds pos (may be pos-3..pos)
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(base_addr + q0);
    uint32_t lo = dm_fmt_ldw<NC>(wp), hi = dm_fmt_ldw<NC>(wp + 1), nx = dm_fmt_ldw<NC>(wp + 2);
    uint32_t found = DM_FMT_NOT_FOUND;
    for (;;) {
        const uint32_t x1 = __funnelshift_r(lo, hi, 8), x2 = __funnelshift_r(lo, hi, 16), x3 = __funnelshift_r(lo, hi, 24);
        uint32_t h = (((lo ^ w0) & m0) == 0 ? 1u : 0u) | (((x1 ^ w0) & m0) == 0 ? 2u : 0u) |
                     (((x2 ^ w0) & m0) == 0 ? 4u : 0u) | (((x3 ^ w0) & m0) == 0 ? 8u : 0u);
        if (q0 < pos) h &= 0xFu << (pos - q0);                                    // positions in front of pos (first word only)
        if (q0 + 3u > last) h &= (last >= q0) ? (0xFu >> (3u - (last - q0))) : 0u;   // positions behind last
        while (h) {
            const uint32_t q = q0 + (uint32_t)__ffs(h) - 1u;
            h &= h - 1;
            bool ok = true;
            for (uint32_t j = 4; j < len; j += 4) {
                const uint32_t lm = len - j >= 4 ? 0xFFFFFFFFu : dm_fmt_tail_mask(len - j);
                if (((dm_fmt_load4<NC>(buf, q + j) ^ lit[j >> 2]) & lm) != 0) { ok = false; break; }
            }
            if (ok) { found = q; break; }
        }
        if (found != DM_FMT_NOT_FOUND || q0 + 4u > last) break;
        q0 += 4;
        lo = hi; hi = nx; ++wp; nx = dm_fmt_ldw<NC>(wp + 2);
    }
    return found;
}

template <bool NC>
__device__ __forceinline__ bool dm_fmtl_match_at(const uint8_t* buf, uint32_t q, const uint32_t* lit, uint32_t len) {
    for (uint32_t j = 0; j < len; j += 4) {
        const uint32_t m = len - j >= 4 ? 0xFFFFFFFFu : dm_fmt_tail_mask(len - j);
        if (((dm_fmt_load4<NC>(buf, q + j) ^ lit[j >> 2]) & m) != 0) return false;
    }
    return true;
}

// One lane matches chain c against text [s, e); needed captures go to caps[slot * DM_FMTL_THREADS]
// (the caller passes its own column).  Returns the number of captures, or 0xFFFFFFFF on mismatch.
// EVERY lane of the warp calls this with the same chain and runs the same number of steps (a lane
// that is inactive or has already failed just idles): the __syncwarp() after each literal is
// what keeps the 32 records of a warp in lockstep -- without it the lanes drift apart through
// the data-dependent search loops and the warp degenerates to 3 active threads per instruction.
template <bool NC>
__device__ uint32_t dm_fmtl_match_chain(const DmFormat& f, uint32_t c, const uint8_t* buf, uint32_t s,
                                        uint32_t e, uint2* caps, bool active) {
    const uint32_t first = f.chain_first[c];
    const uint32_t n = (uint32_t)f.chain_first[c + 1] - first;
    const bool endcap = f.chain_endcap[c] != 0;
    const uint32_t need = f.chain_need[c];
    uint32_t pos = s;
    bool ok = active;
    for (uint32_t i = 0; i < n; ++i) {
        if (ok) {
            const uint32_t len = f.lit_len[first + i];
            const uint32_t* lit = f.pool + f.lit_off[first + i];
            uint32_t q = DM_FMT_NOT_FOUND;
            if (i == 0) {
                if (e >= pos + len && dm_fmtl_match_at<NC>(buf, pos, lit, len)) q = pos;
            } else if (i == n - 1 && !endcap) {
                if (e >= pos + len && dm_fmtl_match_at<NC>(buf, e - len, lit, len)) q = e - len;
            } else {
                q = dm_fmtl_find<NC>(buf, pos, e, lit, len);
            }
            if (q == DM_FMT_NOT_FOUND) {
                ok = false;
            } else {
                if (i > 0 && ((need >> (i - 1)) & 1u))
                    caps[(uint32_t)__popc(need & ((1u << (i - 1)) - 1u)) * DM_FMTL_THREADS] = make_uint2(pos, q - pos);
                pos = q + len;
            }
        }
        __syncwarp();
    }
    if (!ok) return 0xFFFFFFFFu;
    if (endcap) {
        const uint32_t ci = n ? n - 1 : 0;
        const uint32_t cs = n ? pos : s;
        if ((need >> ci) & 1u) caps[(uint32_t)__popc(need & ((1u << ci) - 1u)) * DM_FMTL_THREADS] = make_uint2(cs, e - cs);
        return n ? n : 1;
    }
    if (pos != e) return 0xFFFFFFFFu;
    return n ? n - 1 : 0;
}

// R-norm: text[s, s+len) without the bytes of f.norm_drop, letters folded, written to nbuf at
// the SAME offset (the copy is never longer, so the records of a message cannot collide).
// Aligned words are stored whole; the first and last partial word byte by byte, because the
// rest of those words belongs to a neighbouring record another lane may be writing.
// Returns the normalised length.
__device__ __forceinline__ uint32_t dm_fmtl_normalise(const DmFormat& f, const uint8_t* __restrict__ buf, uint8_t* nbuf,
                                                      uint32_t s, uint32_t len) {
    const bool fold = (f.norm_flags & DM_NORM_LOWERCASE) != 0;
    uint32_t o = s, acc = 0;
    for (uint32_t i = 0; i < len; i += 4) {
        const uint32_t w = dm_fmt_load4(buf, s + i);
        const uint32_t nb = len - i < 4u ? len - i : 4u;
#pragma unroll
        for (uint32_t j = 0; j < 4; ++j) {
            uint32_t c = (w >> (8u * j)) & 0xFFu;
            if (j >= nb || ((f.norm_drop[c >> 5] >> (c & 31u)) & 1u)) continue;
            if (fold && c - 0x41u < 26u) c += 0x20u;
            acc |= c << ((o & 3u) * 8u);
            ++o;
            if ((o & 3u) == 0) {
                if (o - 4u >= s) *reinterpret_cast<uint32_t*>(nbuf + (o - 4u)) = acc;
                else for (uint32_t b = s; b < o; ++b) nbuf[b] = (uint8_t)(acc >> ((b & 3u) * 8u));
                acc = 0;
            }
        }
    }
    const uint32_t w0 = o & ~3u;
    for (uint32_t b = w0 > s ? w0 : s; b < o; ++b) nbuf[b] = (uint8_t)(acc >> ((b & 3u) * 8u));
    return o - s;
}

// Is monitor k present in this record, and where is its value?  Present exactly when the log_format matched (hok), the
// record is in the monitor's event scope, and the header capture exists / the variable index is below the matched
// template's wildcard count.  The value is cap = (offset, length) in `buf` for a header capture and for a variable
// without R-norm; under R-norm a variable is a slice of the normalised copy `nbuf` (see dm_fmtl_value_fp).
__device__ __forceinline__ bool dm_fmtl_locate(const DmFormat& f, uint32_t k, bool hok, int32_t eid, uint32_t n_hcaps,
                                               uint32_t n_vars, const uint2* hcap, const uint2* vcap, uint2& cap) {
    const uint32_t idx = f.mon_index[k];
    bool use = hok && idx != DM_FMT_NONE && !(f.mon_has_event[k] && eid != f.mon_event[k]);
    cap = make_uint2(0, 0);
    if (use) {
        if (f.mon_source[k]) {
            use = eid >= 0 && idx < n_vars;
            if (use) cap = vcap[(uint32_t)__popc(f.chain_need[eid + 1] & ((1u << idx) - 1u)) * DM_FMTL_THREADS];
        } else {
            use = idx < n_hcaps;
            if (use) cap = hcap[(uint32_t)__popc(f.chain_need[0] & ((1u << idx) - 1u)) * DM_FMTL_THREADS];
        }
    }
    return use;
}

// dm_fp64 of the value of monitor k that dm_fmtl_locate found
template <bool NORM>
__device__ __forceinline__ uint64_t dm_fmtl_value_fp(const DmFormat& f, uint32_t k, const uint8_t* buf, const uint8_t* nbuf,
                                                     uint2 cap) {
    return (NORM && f.mon_source[k]) ? dm_fmt_fp64<false>(nbuf, cap.x, cap.y) : dm_fmt_fp64<true>(buf, cap.x, cap.y);
}

// NORM: R-norm is configured; the templates then run on `nbuf`, the per-message normalised copy.
// COMBO: combination monitors (a.combos is a DmMonitors, dm_set_combos; DESIGN.md R-combo): after the single
// monitors, each combination folds the fingerprints of its members, re-hashed from the captures this lane keeps, into
// one key under field n_mons + c.  Member-only monitors are not probed on their own.  (COMBO defaults to false, so
// that `dm_k_format_lanes<TRAIN, NORM>` is the single-monitor kernel it always was.)
template <bool TRAIN, bool NORM, bool COMBO = false>
__global__ void __launch_bounds__(DM_FMTL_THREADS) dm_k_format_lanes(DmDetectArgs a, const DmFormat* __restrict__ gfmt,
                                                                     uint8_t* nbuf) {
    // [2][max_slots][DM_FMTL_THREADS]: header captures, template captures
#ifdef DM_EMU
    uint2* s_caps = reinterpret_cast<uint2*>(g_emu_dyn_smem.data());
#else
    extern __shared__ uint2 s_caps[];
#endif
    __shared__ DmFormat sf;
    __shared__ unsigned int s_unk[DM_MAX_KEYS];
    __shared__ unsigned long long s_anom, s_score, s_bad;
    dm_pdl_wait();                                    // K_A / the training pass are complete (dm_kernels_index.cuh)
    {
        // the grid is sized for the worst case (the record count is only known on the device):
        // CTAs without records leave before touching anything
        const uint64_t n_lines0 = a.hdr_in->n_lines;
        const uint64_t hi0 = a.line_hi < n_lines0 ? a.line_hi : n_lines0;
        if (a.hdr_in->error || a.line_lo + (uint64_t)blockIdx.x * blockDim.x >= hi0) return;
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(gfmt);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sf);
        for (uint32_t i = threadIdx.x; i < sizeof(DmFormat) / 4; i += blockDim.x) dst[i] = src[i];
        if (threadIdx.x < DM_MAX_KEYS) s_unk[threadIdx.x] = 0;
        if (threadIdx.x == 0) { s_anom = 0; s_score = 0; s_bad = 0; }
    }
    __syncthreads();
    if (a.hdr_in->error) return;
    const uint8_t* __restrict__ buf = a.buf;
    const uint32_t tid = threadIdx.x;
    uint2* hcap = s_caps + tid;
    uint2* vcap = s_caps + sf.max_slots * DM_FMTL_THREADS + tid;
    const uint64_t n_lines = a.hdr_in->n_lines;
    const uint64_t hi = a.line_hi < n_lines ? a.line_hi : n_lines;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const DmMonitors* __restrict__ cm = reinterpret_cast<const DmMonitors*>(a.combos);
    const uint32_t member_only = COMBO ? cm->member_only : 0u;

    // the warps iterate a warp-uniform number of times; a lane without a record idles through the
    // same steps (see dm_fmtl_match_chain)
    const uint64_t warp_first = a.line_lo + (uint64_t)blockIdx.x * blockDim.x + (tid & ~31u);
    for (uint64_t wbase = warp_first; wbase < hi; wbase += stride) {
        const uint64_t line = wbase + (tid & 31u);
        const bool act = line < hi;
        const uint32_t s = act ? a.line_start[line] : 0u;
        const uint32_t e = act ? a.line_start[line + 1] - 1 : 0u;
        const uint32_t n_hcaps = dm_fmtl_match_chain<true>(sf, 0, buf, s, e, hcap, act);
        const bool hok = n_hcaps != 0xFFFFFFFFu;
        int32_t eid = -1;
        uint32_t n_vars = 0;
        if (sf.content_capture != DM_FMT_NONE) {
            uint2 cc = make_uint2(0, 0);
            if (hok) cc = hcap[(uint32_t)__popc(sf.chain_need[0] & ((1u << sf.content_capture) - 1u)) * DM_FMTL_THREADS];
            if (NORM) {
                if (hok) cc.y = dm_fmtl_normalise(sf, buf, nbuf, cc.x, cc.y);
                __syncwarp();
            }
            const uint8_t* tbuf = NORM ? nbuf : buf;
            for (uint32_t t = 1; t < sf.n_chains; ++t) {
                const uint32_t nv = dm_fmtl_match_chain<!NORM>(sf, t, tbuf, cc.x, cc.x + cc.y, vcap, hok && eid < 0);
                if (nv != 0xFFFFFFFFu) { eid = (int32_t)t - 1; n_vars = nv; }
            }
        }
        uint32_t unknown = 0;
        for (uint32_t k = 0; k < sf.n_mons; ++k) {
            if (COMBO && ((member_only >> k) & 1u)) continue;                  // (warp-uniform)
            uint2 cap;
            if (dm_fmtl_locate(sf, k, hok, eid, n_hcaps, n_vars, hcap, vcap, cap)) {
                const uint64_t key = dm_make_key(dm_fmtl_value_fp<NORM>(sf, k, buf, nbuf, cap), dm_field_salt(k));
                if (TRAIN) dm_table_insert(a.table, key, &a.hdr->error);
                else if (!dm_table_contains(a.table, key)) unknown |= 1u << k;
            }
            __syncwarp();
        }
        if (COMBO) {
            // combination c = ordered tuple of its members' values; yielded only when every member is present
            for (uint32_t c = 0, n_combos = cm->n_combos; c < n_combos; ++c) {
                const uint32_t lo = cm->combo_off[c], hi_m = cm->combo_off[c + 1];
                uint64_t acc = dm_combo_seed(hi_m - lo);
                bool all = true;
                for (uint32_t j = lo; j < hi_m && all; ++j) {
                    const uint32_t k = cm->combo_members[j];
                    uint2 cap;
                    all = dm_fmtl_locate(sf, k, hok, eid, n_hcaps, n_vars, hcap, vcap, cap);
                    if (all) acc = dm_combo_fold(acc, dm_fmtl_value_fp<NORM>(sf, k, buf, nbuf, cap));
                }
                if (all) {
                    const uint64_t key = dm_make_key(acc ? acc : 1ull, dm_field_salt(sf.n_mons + c));
                    if (TRAIN) dm_table_insert(a.table, key, &a.hdr->error);
                    else if (!dm_table_contains(a.table, key)) unknown |= 1u << (sf.n_mons + c);
                }
                __syncwarp();
            }
        }
        if (!act) continue;
        if (!hok) atomicAdd(&s_bad, 1ull);
        const uint32_t cnt = (uint32_t)__popc(unknown);
        if (line < a.out_cap) {
            if (a.flags) a.flags[line] = cnt ? 1 : 0;
            if (a.scores) a.scores[line] = (float)cnt;
        }
        if (cnt) {
            atomicAdd(&s_anom, 1ull);
            atomicAdd(&s_score, (unsigned long long)cnt);
            uint32_t m = unknown;
            while (m) { const int b = __ffs(m) - 1; m &= m - 1; atomicAdd(&s_unk[b], 1u); }
            const unsigned int at = atomicAdd(&a.hdr->anomaly_list_count, 1u);
            if (at < a.anomaly_cap) {
                dm_anomaly_t r; r.line = (uint32_t)line; r.mask = unknown; r.offset = s;
                a.anomalies[at] = r;
            }
        }
    }
    dm_pdl_launch_dependents();                       // the next step's K_A may start streaming its message in
    __syncthreads();
    if (threadIdx.x == 0 && s_bad) atomicAdd(a.stats + 7, s_bad);
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

// R-norm runs when normalisation is configured and there are templates to run on the normalised Content.
static inline bool dm_format_norm(const DmFormat& f) { return f.norm_flags != 0 && f.n_chains > 1; }

// The instantiation a launch runs.
typedef void (*DmFormatLanesKernel)(DmDetectArgs, const DmFormat*, uint8_t*);
static inline DmFormatLanesKernel dm_format_lanes_kernel(bool train, bool norm, bool combo) {
    if (train) {
        if (norm) return combo ? dm_k_format_lanes<true, true, true> : dm_k_format_lanes<true, true, false>;
        return combo ? dm_k_format_lanes<true, false, true> : dm_k_format_lanes<true, false, false>;
    }
    if (norm) return combo ? dm_k_format_lanes<false, true, true> : dm_k_format_lanes<false, true, false>;
    return combo ? dm_k_format_lanes<false, false, true> : dm_k_format_lanes<false, false, false>;
}
