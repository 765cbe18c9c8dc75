// dm_kernels_parse.cuh -- the MatcherParser stage on the device (rule R-parse, DESIGN.md): LogSchema records in,
// varint-delimited ParserSchemas out.
//
// The host path (parser.py: B200MatcherParser._parse_host, wire.encode_parser_schema) is the specification: for one
// message these kernels write, byte for byte, the ParserSchemas the host writes for it.  Launches, with one host
// readback between the size and the write pass:
//   dm_k_logs_walk / scan / compact   (dm_kernels_logs.cuh) per record its text, and its rank among the usable records
//                                     (rec_line): the j of its parsedLogID
//   dm_k_parse<NORM, false>           one thread per record, DM_FMTL_THREADS per CTA: the header chain, (R-norm) the
//                                     Content normalised into nbuf, the template chains -- the matcher's own dm_fmtl_*
//                                     functions, every capture and wildcard kept -- and the exact size of the record's
//                                     ParserSchema with its length prefix; 0 for a malformed or unusable record
//   dm_alert_scan                     exclusive scan of the sizes: where each ParserSchema goes; the total
//   dm_k_parse<NORM, true>            the same match again, then each warp writes its 32 records one after another:
//                                     lane 0 the tags and varints, all 32 lanes the spans and constants, consecutive
//                                     bytes per lane
#pragma once
#include "dm_device.cuh"
#include "dm_kernels_logs.cuh"
#include "dm_kernels_format.cuh"

#define DMP_POOL 65536                             // bytes of constant text: fields 1-3, template texts, capture names

// What dm_set_parser_format fixes: everything of a ParserSchema that does not depend on the record or the call.
struct DmParseFmt {
    uint32_t head_len;                             // pool[0, head_len): fields 1-3, tags and lengths included
    uint32_t n_templates;
    uint32_t tmpl_off[DM_FMT_MAX_CHAINS], tmpl_len[DM_FMT_MAX_CHAINS];    // template text t, verbatim
    uint32_t n_names;                              // header captures = logFormatVariables keys, in output order
    uint32_t name_off[DM_FMT_MAX_CAPTURES], name_len[DM_FMT_MAX_CAPTURES];
    uint32_t name_cap[DM_FMT_MAX_CAPTURES];        //   and the capture each one names
    uint8_t pool[DMP_POOL];
};

struct DmParseArgs {
    const DmParseFmt* pf;
    const DmFormat* pfmt;                          // the matcher's format keeping every capture (dm_parse_efmt_build)
    const uint8_t* buf;                            // the caller's message
    uint8_t* nbuf;                                 // R-norm: the message-sized scratch the Content is normalised into
    uint32_t n_records;
    const uint32_t* rec_off;                       // per record: its payload (dm_kernels_logs.cuh)
    const uint32_t* rec_len;
    const uint32_t* text_off;                      //   its text, DML_UNUSABLE length if it has none
    const uint32_t* text_len;
    const uint32_t* rank;                          //   its rank among the usable records (rec_line)
    unsigned long long* size;                      //   bytes of its ParserSchema, then where it goes
    long long first_id;                            // parsedLogID of the first record emitted
    long long now;                                 // receivedTimestamp = parsedTimestamp
    uint8_t* out;
    unsigned long long out_cap;
    const unsigned long long* total;               // written by the scan; the write pass checks it against out_cap
};

// Bytes go to o[n] when o is set, otherwise they are only counted.  In the write pass every lane of a warp runs the same
// field sequence on the same record: lane 0 stores the single bytes, the 32 lanes share the spans.
struct DmpOut {
    uint8_t* o;
    unsigned long long n;
    uint32_t lane;
    __device__ __forceinline__ void byte(uint8_t c) { if (o && lane == 0) o[n] = c; ++n; }
    __device__ __forceinline__ void span(const uint8_t* p, uint32_t len) {
        if (o) for (uint32_t i = lane; i < len; i += 32) o[n + i] = p[i];
        n += len;
    }
    __device__ __forceinline__ void varint(unsigned long long v) {
        while (v >= 0x80u) { byte((uint8_t)(v | 0x80u)); v >>= 7; }
        byte((uint8_t)v);
    }
    __device__ __forceinline__ void str(uint8_t tag, const uint8_t* p, uint32_t len) { byte(tag); varint(len); span(p, len); }
};

__device__ __forceinline__ uint32_t dmp_varint_len(unsigned long long v) {
    uint32_t k = 1;
    while (v >= 0x80u) { v >>= 7; ++k; }
    return k;
}

// One record as its ParserSchema needs it.  Captures are (offset, length) in buf; variables in nbuf under R-norm.
struct DmpRec {
    uint32_t tp, tl;                               // the text
    uint32_t lp, ll;                               // logID: the last field 2 of the payload, ll = 0 when it has none
    int32_t eid;
    uint32_t n_vars;
    bool hok;                                      // the log_format matched: logFormatVariables are written
    uint32_t rank;
    const uint2* hcap;                             // capture c at hcap[c * DM_FMTL_THREADS]
    const uint2* vcap;                             // variable v at vcap[v * DM_FMTL_THREADS]
};

// The ParserSchema of one record without its length prefix, in wire.encode_parser_schema's field order.
__device__ __forceinline__ void dmp_body(DmpOut& w, const DmParseArgs& a, const DmParseFmt& P, const DmpRec& R,
                                         const uint8_t* vbuf) {
    w.span(P.pool, P.head_len);                                      // 1 __version__, 2 parserType, 3 parserID
    w.byte(0x20);                                                    // 4 EventID (a negative int32 takes 10 bytes)
    w.varint((unsigned long long)(long long)R.eid);
    if (R.eid >= 0) w.str(0x2A, P.pool + P.tmpl_off[R.eid], P.tmpl_len[R.eid]);       // 5 template
    for (uint32_t v = 0; v < R.n_vars; ++v) {                        // 6 variables
        const uint2 c = R.vcap[v * DM_FMTL_THREADS];
        w.str(0x32, vbuf + c.x, c.y);
    }
    {                                                                // 7 parsedLogID = str(first_id + rank)
        const long long id = a.first_id + (long long)R.rank;
        unsigned long long m = id < 0 ? 0ull - (unsigned long long)id : (unsigned long long)id;
        uint8_t d[20];
        uint32_t k = 0;
        do { d[k++] = (uint8_t)('0' + m % 10u); m /= 10u; } while (m);
        w.byte(0x3A);
        w.varint(k + (id < 0 ? 1u : 0u));
        if (id < 0) w.byte('-');
        while (k) w.byte(d[--k]);
    }
    w.str(0x42, a.buf + R.lp, R.ll);                                 // 8 logID
    w.str(0x4A, a.buf + R.tp, R.tl);                                 // 9 log
    if (R.hok) {
        for (uint32_t j = 0; j < P.n_names; ++j) {                   // 10 logFormatVariables, in key order
            const uint2 c = R.hcap[P.name_cap[j] * DM_FMTL_THREADS];
            const uint32_t kl = P.name_len[j];
            w.byte(0x52);
            w.varint(1 + dmp_varint_len(kl) + kl + 1 + dmp_varint_len(c.y) + c.y);
            w.str(0x0A, P.pool + P.name_off[j], kl);
            w.str(0x12, a.buf + c.x, c.y);
        }
    }
    w.byte(0x58);                                                    // 11 receivedTimestamp
    w.varint((unsigned long long)a.now);
    w.byte(0x60);                                                    // 12 parsedTimestamp
    w.varint((unsigned long long)a.now);
}

// logID of a LogSchema payload [pos, end) that dm_pb_walk_log accepted: its last field 2 (LEN), empty when absent.
__device__ __forceinline__ void dmp_log_id(const uint8_t* buf, uint32_t pos, uint32_t end, uint32_t& lp, uint32_t& ll) {
    lp = pos;
    ll = 0;
    while (pos < end) {
        uint32_t field, wt;
        if (!dm_pb_tag(buf, pos, end, field, wt)) return;
        if (wt != 2) {
            if (!dm_pb_skip(buf, pos, end, wt)) return;
            continue;
        }
        uint64_t len;
        if (!dm_pb_varint(buf, pos, end, len) || len > (uint64_t)(end - pos)) return;
        if (field == 2) { lp = pos; ll = (uint32_t)len; }
        pos += (uint32_t)len;
    }
}

// NORM: R-norm runs (dm_format_norm).  !WRITE: the size pass; WRITE: the write pass.  The warps iterate a warp-uniform
// number of times and a lane without a usable record idles through the same steps (see dm_fmtl_match_chain).
template <bool NORM, bool WRITE>
__global__ void __launch_bounds__(DM_FMTL_THREADS) dm_k_parse(DmParseArgs a) {
#ifdef DM_EMU
    uint2* s_caps = reinterpret_cast<uint2*>(g_emu_dyn_smem.data());
#else
    extern __shared__ uint2 s_caps[];
#endif
    const DmFormat& f = *a.pfmt;
    const DmParseFmt& P = *a.pf;
    if (WRITE && *a.total > a.out_cap) return;                      // (the host grows the buffer before this launch)
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    uint2* hcap = s_caps + tid;
    uint2* vcap = s_caps + f.max_slots * DM_FMTL_THREADS + tid;
    const uint8_t* vbuf = NORM ? a.nbuf : a.buf;
    for (uint32_t wbase = blockIdx.x * blockDim.x + (tid & ~31u); wbase < a.n_records; wbase += gridDim.x * blockDim.x) {
        const uint32_t r = wbase + lane;
        const bool act = r < a.n_records && a.text_len[r] != DML_UNUSABLE;
        const uint32_t s = act ? a.text_off[r] : 0u;
        const uint32_t e = act ? s + a.text_len[r] : 0u;
        const uint32_t n_hcaps = dm_fmtl_match_chain<true>(f, 0, a.buf, s, e, hcap, act);
        const bool hok = n_hcaps != 0xFFFFFFFFu;
        int32_t eid = -1;
        uint32_t n_vars = 0;
        if (f.content_capture != DM_FMT_NONE) {
            uint2 cc = make_uint2(0, 0);
            if (hok) cc = hcap[f.content_capture * DM_FMTL_THREADS];
            if (NORM) {
                if (hok) cc.y = dm_fmtl_normalise(f, a.buf, a.nbuf, cc.x, cc.y);
                __syncwarp();
            }
            for (uint32_t t = 1; t < f.n_chains; ++t) {
                const uint32_t nv = dm_fmtl_match_chain<!NORM>(f, t, vbuf, cc.x, cc.x + cc.y, vcap, hok && eid < 0);
                if (nv != 0xFFFFFFFFu) { eid = (int32_t)t - 1; n_vars = nv; }
            }
        }
        DmpRec R;
        R.tp = s; R.tl = e - s; R.eid = eid; R.n_vars = n_vars; R.hok = hok;
        R.lp = 0; R.ll = 0; R.rank = 0;
        if (act) {
            dmp_log_id(a.buf, a.rec_off[r], a.rec_off[r] + a.rec_len[r], R.lp, R.ll);
            R.rank = a.rank[r];
        }
        if (!WRITE) {
            if (r < a.n_records) {
                unsigned long long bytes = 0;
                if (act) {
                    R.hcap = hcap; R.vcap = vcap;
                    DmpOut c{nullptr, 0, 0};
                    dmp_body(c, a, P, R, vbuf);
                    bytes = dmp_varint_len(c.n) + c.n;
                }
                a.size[r] = bytes;
            }
            continue;
        }
        const unsigned long long at = act ? a.size[r] : 0ull;
        __syncwarp();                                                // (the other lanes read this lane's captures and nbuf)
        const uint32_t wbase_tid = tid & ~31u;
        for (uint32_t i = 0; i < 32; ++i) {
            if (!__shfl_sync(0xffffffffu, (int)act, i)) continue;   // (warp-uniform)
            DmpRec Q;
            Q.tp = __shfl_sync(0xffffffffu, R.tp, i);
            Q.tl = __shfl_sync(0xffffffffu, R.tl, i);
            Q.lp = __shfl_sync(0xffffffffu, R.lp, i);
            Q.ll = __shfl_sync(0xffffffffu, R.ll, i);
            Q.eid = __shfl_sync(0xffffffffu, R.eid, i);
            Q.n_vars = __shfl_sync(0xffffffffu, R.n_vars, i);
            Q.hok = __shfl_sync(0xffffffffu, (int)R.hok, i) != 0;
            Q.rank = __shfl_sync(0xffffffffu, R.rank, i);
            Q.hcap = s_caps + wbase_tid + i;
            Q.vcap = s_caps + f.max_slots * DM_FMTL_THREADS + wbase_tid + i;
            DmpOut c{nullptr, 0, 0};
            dmp_body(c, a, P, Q, vbuf);
            DmpOut w{a.out, __shfl_sync(0xffffffffu, at, i), lane};
            w.varint(c.n);
            dmp_body(w, a, P, Q, vbuf);
        }
        __syncwarp();                                                // (before the next round overwrites the captures)
    }
}

typedef void (*DmParseKernel)(DmParseArgs);
static inline DmParseKernel dm_parse_kernel(bool norm, bool write) {
    if (norm) return write ? dm_k_parse<true, true> : dm_k_parse<true, false>;
    return write ? dm_k_parse<false, true> : dm_k_parse<false, false>;
}

// ---------------------------------------------------------------------------------------------- host side
// The matcher's format as the parser needs it: chain 0 keeps every capture and every template every wildcard, so that
// capture c and variable v sit in slot c and v.
static inline void dm_parse_efmt_build(const DmFormat& f, DmFormat* out) {
    *out = f;
    out->max_slots = 1;
    for (uint32_t c = 0; c < out->n_chains; ++c) {
        const uint32_t lits = (uint32_t)out->chain_first[c + 1] - out->chain_first[c];
        const uint32_t caps = out->chain_endcap[c] ? lits : (lits ? lits - 1 : 0);
        out->chain_need[c] = caps >= 32 ? 0xFFFFFFFFu : (1u << caps) - 1u;
        if (caps > out->max_slots) out->max_slots = caps;
    }
}

// Fills P from the handle's format f and dm_set_parser_format's arguments: strings = __version__, parserType, parserID,
// the templates in EventID order, then the capture names in output order; name j is capture capture_order[j].  Returns
// nullptr or the reason the arguments are refused.
static inline const char* dm_parse_fmt_build(const DmFormat& f, uint32_t n_strings, const uint8_t* blob, const uint32_t* lens,
                                             const uint32_t* capture_order, DmParseFmt* P) {
    memset(P, 0, sizeof(*P));
    const uint32_t n_templates = f.n_chains ? f.n_chains - 1 : 0;
    const uint32_t lits = f.n_chains ? (uint32_t)f.chain_first[1] - f.chain_first[0] : 0;
    const uint32_t n_caps = f.n_chains ? (f.chain_endcap[0] ? lits : (lits ? lits - 1 : 0)) : 0;
    if (n_strings != 3 + n_templates + n_caps) return "n_strings must be 3 + templates + captures of the log_format";
    if (n_caps && !capture_order) return "capture_order is NULL";
    uint32_t seen = 0;
    for (uint32_t j = 0; j < n_caps; ++j) {
        if (capture_order[j] >= n_caps || (seen >> capture_order[j] & 1u)) return "capture_order is not a permutation of the captures";
        seen |= 1u << capture_order[j];
    }
    uint64_t pos = 0, src = 0;
    auto put = [&](const uint8_t* p, uint64_t n) -> bool {
        if (pos + n > DMP_POOL) return false;
        memcpy(P->pool + pos, p, n);
        pos += n;
        return true;
    };
    const uint8_t tags[3] = {0x0A, 0x12, 0x1A};
    for (uint32_t i = 0; i < 3; ++i) {
        uint8_t hdr[11];
        int k = 0;
        hdr[k++] = tags[i];
        uint64_t v = lens[i];
        while (v >= 0x80u) { hdr[k++] = (uint8_t)(v | 0x80u); v >>= 7; }
        hdr[k++] = (uint8_t)v;
        if (!put(hdr, k) || !put(blob + src, lens[i])) return "the strings exceed 64 KiB";
        src += lens[i];
    }
    P->head_len = (uint32_t)pos;
    P->n_templates = n_templates;
    for (uint32_t t = 0; t < n_templates; ++t) {
        P->tmpl_off[t] = (uint32_t)pos;
        P->tmpl_len[t] = lens[3 + t];
        if (!put(blob + src, lens[3 + t])) return "the strings exceed 64 KiB";
        src += lens[3 + t];
    }
    P->n_names = n_caps;
    for (uint32_t j = 0; j < n_caps; ++j) {
        P->name_off[j] = (uint32_t)pos;
        P->name_len[j] = lens[3 + n_templates + j];
        P->name_cap[j] = capture_order[j];
        if (!put(blob + src, P->name_len[j])) return "the strings exceed 64 KiB";
        src += P->name_len[j];
    }
    return nullptr;
}
