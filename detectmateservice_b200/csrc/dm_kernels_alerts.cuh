// dm_kernels_alerts.cuh -- the DetectorSchema alerts of the last batch, encoded on the device (rule R-alert, DESIGN.md).
//
// The host path (component.py: _process_lines_one / _process_logs / _process_record_batch, _detector_schema,
// wire.encode_detector_schema) is the specification: for the last dm_process_lines, dm_process_logs or
// dm_process_records batch these kernels write, byte for byte, the varint-delimited DetectorSchemas the host writes for
// it.  Launches for raw lines, with no host round trip in between:
//   dm_k_alert_mark     one thread per anomaly entry: mark its record
//   dm_alert_scan       exclusive scan of the marks: the rank of each anomalous record, in record order; the count
//   dm_k_alert_gather   one thread per anomaly entry: OR its mask into its record's merged mask (the stream kernel appends
//                       one entry per unknown field, in no particular order)
//   dm_k_alert_size     one thread per anomalous record: the R-tok scan of the record and the bytes of its DetectorSchema;
//                       a record the device cannot word exactly (its Time string is outside the grammar) declines
//   dm_alert_scan       exclusive scan of the sizes: where each DetectorSchema goes; the total
//   dm_k_alert_write    one thread per anomalous record: the same walk as dm_k_alert_size, writing
// In log_format mode dm_k_alert_format (NORM, !WRITE / WRITE) takes the place of the size / write kernels: it re-runs the
// header and template chains with the matcher's own device functions (dm_fmtl_*, dm_kernels_format.cuh) before the walk.
// LogSchema batches (DMA_LOGS) take the same launches: dm_k_logs_scatter has already rewritten the anomaly list to
// record indices, and a record's text is its line of the compacted buffer, so only dm_k_alert_gather (where the text
// starts) and the logID (the last field 2 of the payload, dma_log_id) differ.  ParserSchema batches (DMA_RECORDS) have
// no anomaly list: dm_k_alert_mark_records / dm_k_alert_gather_records take the per-record flags and masks, and
// dm_k_alert_records<false / true> walks each anomalous record once with the detection kernels' own walk.
// A record is walked by one thread; a record of max_batch_bytes is walked by one thread too, slowly but correctly.
#pragma once
#include "dm_device.cuh"
#include "dm_kernels_records.cuh"
#include "dm_kernels_format.cuh"

#define DMA_THREADS 256
#define DMA_ITEMS 16                               // scan: elements per thread
#define DMA_TILE (DMA_THREADS * DMA_ITEMS)
#define DMA_POOL 16384                             // bytes of constant text (fields 1-3, field 10, alert keys)
#define DMA_MSG DM_MAX_KEYS                        // key slot of "msg", the Time source of R-tok L7
#define DMA_NONE 0xFFu
#define DMA_LINES 0u                               // DmAlertArgs::src: the batch came from dm_process_lines,
#define DMA_LOGS 1u                                //   dm_process_logs
#define DMA_RECORDS 2u                             //   or dm_process_records
#define DMA_SRC_NONE 0xFFu                         //   or none of them: there is nothing to word

// What dm_set_alert_format fixes: everything of a DetectorSchema that does not depend on the record or the call.
struct DmAlertFmt {
    uint32_t n_keys;                               // monitors: mask bit k < n_keys = monitor k
    uint32_t n_out;                                // alert keys, in output order (UTF-8 byte order, as the host sorts)
    uint32_t key_len[DM_MAX_KEYS + 1];             // R-tok key of monitor k; [DMA_MSG] = "msg"
    uint8_t key[DM_MAX_KEYS + 1][DM_MAX_KEYLEN];
    uint32_t out_off[DM_MAX_KEYS], out_len[DM_MAX_KEYS];   // alert key j = pool[out_off[j], + out_len[j])
    uint32_t sup_off[DM_MAX_KEYS + 1];             // mask bits supplying alert key j: sup[sup_off[j], sup_off[j + 1]),
    uint8_t sup[DM_MAX_KEYS];                      //   in config order (the last one set wins, as in a dict comprehension)
    uint32_t n_combos;                             // combination c = mask bit n_keys + c, of the monitors
    uint32_t combo_off[DM_MAX_KEYS + 1];           //   members[combo_off[c], combo_off[c + 1])
    uint8_t members[DM_MAX_COMBO_MEMBERS];
    uint32_t time_cap;                             // log_format mode: the header capture named Time, DMA_NONE if none
    uint32_t head_len;                             // pool[0, head_len): fields 1-3, tags and lengths included
    uint32_t desc_off, desc_len;                   // field 10, tag and length included
    uint8_t pool[DMA_POOL];
};

// Written by the kernels; the host reads it back with one copy.
struct DmAlertHeader {
    unsigned int n_alerts;                         // anomalous records of the batch = DetectorSchemas
    unsigned int declined;                         // non-zero: a record the device cannot word exactly
    unsigned long long total;                      // bytes of the varint-delimited DetectorSchemas
};

struct DmAlertArgs {
    const DmAlertFmt* fmt;
    const uint8_t* buf;                            // the batch, as dm_process_lines read it
    uint64_t nbytes;
    const float* scores;                           // per record
    const dm_anomaly_t* anoms;                     // the anomaly list of the batch
    uint32_t n_entries;                            // its entries (at most the list's capacity)
    uint64_t n_lines;
    uint32_t* rank;                                // per record + 1: mark, then its rank among the anomalous records
    uint32_t* rec_line;                            // per anomalous record: record index
    uint32_t* rec_mask;                            //   merged mask (zeroed before dm_k_alert_gather)
    unsigned long long* rec_off;                   //   offset of its first byte
    unsigned long long* size;                      //   bytes of its DetectorSchema, then where it goes
    DmAlertHeader* ahdr;
    unsigned long long first_log_id;               // logID of record 0 (n_seen before the batch)
    long long first_alert_id;                      // alertID of the first anomalous record (start_id + n_alerts)
    long long now;                                 // detectionTimestamp = receivedTimestamp = the fallback Time
    uint8_t* out;
    unsigned long long out_cap;
    const DmFormat* efmt;                          // log_format mode: the matcher's format, keeping the Time capture too
    uint8_t* nbuf;                                 //   R-norm: the message-sized scratch the Content is normalised into
    uint32_t src = DMA_LINES;                      // the batch's input; for DMA_LOGS buf is the compacted texts, scores
                                                   // and anomaly lines are per record
    const uint8_t* pay = nullptr;                  // DMA_LOGS / DMA_RECORDS: the caller's message; per record the offset
    const uint32_t* pay_off = nullptr;             //   and length of its payload
    const uint32_t* pay_len = nullptr;
    const uint32_t* log_line = nullptr;            // DMA_LOGS: per record its line of buf, per line where it starts
    const uint32_t* log_dst = nullptr;
    const uint8_t* flags = nullptr;                // DMA_RECORDS: per record its flag and mask, and the monitors
    const uint32_t* masks = nullptr;
    const DmMonitors* mons = nullptr;
};

// ---------------------------------------------------------------------------------------------- exclusive scan
// In place over d[0, n); the sum goes to *total.  Three launches: tile sums, one CTA over the tile sums, tiles again.
template <typename T>
__device__ __forceinline__ T dma_cta_scan(T v, T* s_warp, T& total) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T x = v;
    for (unsigned d = 1; d < 32; d <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        T w = lane < DMA_THREADS / 32 ? s_warp[lane] : (T)0;
        for (unsigned d = 1; d < 32; d <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += y;
        }
        if (lane < DMA_THREADS / 32) s_warp[lane] = w;
    }
    __syncthreads();
    total = s_warp[DMA_THREADS / 32 - 1];
    const T ex = (warp ? s_warp[warp - 1] : (T)0) + x - v;
    __syncthreads();
    return ex;
}

template <typename T>
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_scan_tiles(const T* d, uint64_t n, T* tile_sums) {
    __shared__ T s_warp[DMA_THREADS / 32];
    const uint64_t base = (uint64_t)blockIdx.x * DMA_TILE + (uint64_t)threadIdx.x * DMA_ITEMS;
    T v = 0;
    for (uint32_t i = 0; i < DMA_ITEMS; ++i)
        if (base + i < n) v += d[base + i];
    T tot;
    dma_cta_scan(v, s_warp, tot);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = tot;
}

template <typename T>
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_scan_top(T* tile_sums, uint32_t n_tiles, T* total) {
    __shared__ T s_warp[DMA_THREADS / 32];
    T carry = 0;
    for (uint32_t b = 0; b < n_tiles; b += DMA_THREADS) {
        const uint32_t t = b + threadIdx.x;
        const T v = t < n_tiles ? tile_sums[t] : (T)0;
        T tot;
        const T ex = dma_cta_scan(v, s_warp, tot);
        if (t < n_tiles) tile_sums[t] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

template <typename T>
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_scan_apply(T* d, uint64_t n, const T* tile_sums) {
    __shared__ T s_warp[DMA_THREADS / 32];
    const uint64_t base = (uint64_t)blockIdx.x * DMA_TILE + (uint64_t)threadIdx.x * DMA_ITEMS;
    T v[DMA_ITEMS];
    T sum = 0;
    for (uint32_t i = 0; i < DMA_ITEMS; ++i) {
        v[i] = base + i < n ? d[base + i] : (T)0;
        sum += v[i];
    }
    T tot;
    T run = tile_sums[blockIdx.x] + dma_cta_scan(sum, s_warp, tot);
    for (uint32_t i = 0; i < DMA_ITEMS; ++i) {
        if (base + i < n) d[base + i] = run;
        run += v[i];
    }
}

// ---------------------------------------------------------------------------------------------- order and merge
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_mark(DmAlertArgs a) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_entries; i += gridDim.x * blockDim.x) {
        const uint32_t line = a.anoms[i].line;
        if (line < a.n_lines) a.rank[line] = 1u;
    }
}

__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_gather(DmAlertArgs a) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_entries; i += gridDim.x * blockDim.x) {
        const dm_anomaly_t e = a.anoms[i];
        if (e.line >= a.n_lines) continue;
        const uint32_t r = a.rank[e.line];
        atomicOr(&a.rec_mask[r], e.mask);
        a.rec_line[r] = e.line;                    // (every entry of a record carries the same line and offset)
        a.rec_off[r] = a.src == DMA_LOGS ? a.log_dst[a.log_line[e.line]] : e.offset;
    }
}

// ParserSchema batches: the flags of dm_process_records mark the anomalous records, their masks are already merged.
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_mark_records(DmAlertArgs a) {
    for (uint64_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_lines; r += gridDim.x * blockDim.x)
        a.rank[r] = a.flags[r] ? 1u : 0u;
}

__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_gather_records(DmAlertArgs a) {
    for (uint64_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_lines; r += gridDim.x * blockDim.x) {
        if (!a.flags[r]) continue;
        const uint32_t k = a.rank[r];
        if (k >= a.n_entries) { atomicOr(&a.ahdr->declined, 1u); continue; }     // (the host sized n_entries from the count)
        a.rec_line[k] = (uint32_t)r;
        a.rec_mask[k] = a.masks[r];
        a.rec_off[k] = a.pay_off[r];
    }
}

// ---------------------------------------------------------------------------------------------- one DetectorSchema
// Bytes go to o[n] when o is set; otherwise they are only counted, so that the size and the write pass are one walk.
struct DmaOut {
    uint8_t* o;
    unsigned long long n;
    __device__ __forceinline__ void byte(uint8_t c) { if (o) o[n] = c; ++n; }
    __device__ __forceinline__ void bytes(const uint8_t* p, uint32_t len) {
        if (o) for (uint32_t i = 0; i < len; ++i) o[n + i] = p[i];
        n += len;
    }
    __device__ __forceinline__ void varint(unsigned long long v) {
        while (v >= 0x80u) { byte((uint8_t)(v | 0x80u)); v >>= 7; }
        byte((uint8_t)v);
    }
    __device__ __forceinline__ void dec(unsigned long long v) {      // decimal digits, as str() of the int
        uint8_t d[20];
        int k = 0;
        do { d[k++] = (uint8_t)('0' + v % 10u); v /= 10u; } while (v);
        while (k) byte(d[--k]);
    }
};

__device__ __forceinline__ uint32_t dma_varint_len(unsigned long long v) {
    uint32_t k = 1;
    while (v >= 0x80u) { v >>= 7; ++k; }
    return k;
}

__device__ __forceinline__ uint32_t dma_dec_len(unsigned long long v) {
    uint32_t k = 1;
    while (v >= 10u) { v /= 10u; ++k; }
    return k;
}

// v.decode("utf-8", "replace").encode("utf-8"): well-formed sequences are copied, every maximal ill-formed subpart
// (the lead byte and the continuation bytes that may still follow it) becomes one U+FFFD, as CPython's decoder does.
__device__ __forceinline__ void dma_utf8_replace(DmaOut& w, const uint8_t* s, uint32_t n) {
    uint32_t i = 0;
    while (i < n) {
        const uint8_t c = s[i];
        if (c < 0x80u) { w.byte(c); ++i; continue; }
        uint32_t need = 0;
        uint8_t lo = 0x80u, hi = 0xBFu;                              // range of the second byte
        if (c >= 0xC2u && c <= 0xDFu) need = 1;
        else if (c >= 0xE0u && c <= 0xEFu) { need = 2; if (c == 0xE0u) lo = 0xA0u; else if (c == 0xEDu) hi = 0x9Fu; }
        else if (c >= 0xF0u && c <= 0xF4u) { need = 3; if (c == 0xF0u) lo = 0x90u; else if (c == 0xF4u) hi = 0x8Fu; }
        uint32_t k = 1;
        while (k <= need && i + k < n) {
            const uint8_t d = s[i + k];
            if (d < (k == 1 ? lo : 0x80u) || d > (k == 1 ? hi : 0xBFu)) break;
            ++k;
        }
        if (need && k == need + 1) w.bytes(s + i, k);
        else { w.byte(0xEFu); w.byte(0xBFu); w.byte(0xBDu); }
        i += k;
    }
}

struct DmaSpan { uint32_t b, e, nrm; };                 // nrm: a slice of the normalised Content, not of the record

__device__ __forceinline__ int dma_lowbit(unsigned long long m) {
    return (uint32_t)m ? __ffs((unsigned)m) - 1 : 31 + __ffs((unsigned)(m >> 32));
}

// First values of the key slots in `want` (R-tok L2-L6), exactly as the host's alerts.record_fields finds them: a key
// starts at the record's first byte or after ' ' or '\'' outside double quotes, runs to the first '=' before any of
// ' ', '"', '\''; its value runs to the first ' ' outside double quotes.  Returns the slots found.
__device__ __forceinline__ unsigned long long dma_fields(const DmAlertFmt& F, const uint8_t* s, uint32_t n,
                                                         unsigned long long want, DmaSpan* span) {
    unsigned long long found = 0;
    bool inq = false;
    for (uint32_t p = 0; p < n && found != want; ++p) {
        const uint8_t c = s[p];
        if (!inq && (p == 0 || s[p - 1] == 0x20u || s[p - 1] == 0x27u)) {
            uint32_t q = p;
            while (q < n && s[q] != 0x3Du && s[q] != 0x20u && s[q] != 0x22u && s[q] != 0x27u) ++q;
            if (q < n && s[q] == 0x3Du && q > p) {
                const uint32_t len = q - p;
                bool have_end = false;
                uint32_t e = q + 1;
                for (unsigned long long m = want & ~found; m; m &= m - 1) {
                    const int k = dma_lowbit(m);
                    if (F.key_len[k] != len) continue;
                    bool eq = true;
                    for (uint32_t i = 0; i < len && eq; ++i) eq = F.key[k][i] == s[p + i];
                    if (!eq) continue;
                    if (!have_end) {
                        bool vq = false;
                        while (e < n && !(s[e] == 0x20u && !vq)) { if (s[e] == 0x22u) vq = !vq; ++e; }
                        have_end = true;
                    }
                    span[k].b = q + 1;
                    span[k].e = e;
                    span[k].nrm = 0;
                    found |= 1ull << k;
                }
            }
        }
        if (c == 0x22u) inq = !inq;
    }
    return found;
}

// extractedTimestamps[0] of Time bytes s, as the host's `int(float(s))` with `now` on ValueError, where the device can
// prove the result: for s in the grammar [0-9]{1,10}(\.[0-9]{0,6})? the integer part (below 2^34 doubles are spaced at
// most 2^-19 apart, less than twice the 1e-6 that separates a 6-digit fraction from the next integer, so the correctly
// rounded float of s never reaches it); `now` for an empty s and for an s holding a byte no float literal can hold
// (CPython's float() of bytes accepts only ASCII white space, digits, '.', '+', '-', 'e', '_' and the letters of inf,
// infinity and nan, in either case).  False for every other string: the record declines.
// str: s is the UTF-8 of a str (a ParserSchema map value), and float() of a str also takes Unicode decimal digits and
// white space.  An ASCII byte outside the alphabet above still proves `now` (every other character maps to one that
// fails the parse), but a string without one that holds a byte >= 0x80 declines.
__device__ __forceinline__ bool dma_time(const uint8_t* s, uint32_t n, long long now, long long* ts, bool str = false) {
    bool foreign = n == 0, wide = false;
    for (uint32_t j = 0; j < n && !foreign; ++j) {
        if (str && s[j] >= 0x80u) { wide = true; continue; }
        const uint8_t c = s[j] | ((s[j] >= 'A' && s[j] <= 'Z') ? 0x20u : 0u);
        foreign = !((c >= '0' && c <= '9') || c == '.' || c == '+' || c == '-' || c == '_' || c == ' ' ||
                    (c >= 0x09u && c <= 0x0Du) || c == 'e' || c == 'i' || c == 'n' || c == 'f' || c == 't' ||
                    c == 'y' || c == 'a');
    }
    if (foreign) { *ts = now; return true; }
    if (wide) return false;
    uint32_t i = 0;
    long long v = 0;
    while (i < n && s[i] >= '0' && s[i] <= '9') { v = v * 10 + (s[i] - '0'); ++i; if (i > 10) return false; }
    if (i == 0) return false;
    if (i < n) {
        if (s[i] != '.' || n - i - 1 > 6) return false;
        for (uint32_t j = i + 1; j < n; ++j)
            if (s[j] < '0' || s[j] > '9') return false;
    }
    *ts = v;
    return true;
}

// One anomalous record as its DetectorSchema needs it.
struct DmaRec {
    const uint8_t* s;                              // base of the value spans: the record (key=value), the message
    const uint8_t* ns;                             //   (log_format) or, for spans marked nrm, the normalised copy
    uint32_t line;
    unsigned long long found;                      // key slots found, and their values
    DmaSpan span[DM_MAX_KEYS + 1];
    uint8_t pick[DM_MAX_KEYS];                     // per alert key: the mask bit that supplies it, DMA_NONE if absent
    long long ts;                                  // extractedTimestamps[0]
    const uint8_t* lid;                            // logIDs[0]: [lid, + lid_n) (LogSchema, ParserSchema), or nullptr:
    uint32_t lid_n;                                //   the decimal first_log_id + line (raw lines)
};

__device__ __forceinline__ void dma_value(DmaOut& w, const DmaRec& R, uint32_t k) {
    if (R.found >> k & 1ull) dma_utf8_replace(w, (R.span[k].nrm ? R.ns : R.s) + R.span[k].b, R.span[k].e - R.span[k].b);
}

// The DetectorSchema text of alert key j's value: "Unknown value: '<v>'" for a monitor, "Unknown value combination:
// ('<v1>', '<v2>')" for a combination.
__device__ __forceinline__ void dma_text(DmaOut& w, const DmAlertFmt& F, const DmaRec& R, uint32_t bit) {
    const uint8_t* one = (const uint8_t*)"Unknown value: '";
    const uint8_t* many = (const uint8_t*)"Unknown value combination: (";
    if (bit < F.n_keys) {
        w.bytes(one, 16);
        dma_value(w, R, bit);
        w.byte('\'');
        return;
    }
    const uint32_t c = bit - F.n_keys;
    w.bytes(many, 28);
    for (uint32_t j = F.combo_off[c]; j < F.combo_off[c + 1]; ++j) {
        const uint32_t m = F.members[j];
        if (j > F.combo_off[c]) { w.byte(','); w.byte(' '); }
        w.byte('\'');
        dma_value(w, R, m);
        w.byte('\'');
    }
    w.byte(')');
}

// The DetectorSchema of one record, without its length prefix, in wire.encode_detector_schema's field order.
__device__ __forceinline__ void dma_body(DmaOut& x, const DmAlertArgs& a, const DmaRec& R, uint32_t r) {
    const DmAlertFmt& F = *a.fmt;
    const long long aid = a.first_alert_id + (long long)r;
    const unsigned long long aid_mag = aid < 0 ? 0ull - (unsigned long long)aid : (unsigned long long)aid;
    x.bytes(F.pool, F.head_len);                                     // 1 __version__, 2 detectorID, 3 detectorType
    x.byte(0x22);                                                    // 4 alertID
    x.varint(dma_dec_len(aid_mag) + (aid < 0 ? 1u : 0u));
    if (aid < 0) x.byte('-');
    x.dec(aid_mag);
    x.byte(0x28);                                                    // 5 detectionTimestamp
    x.varint((unsigned long long)a.now);
    x.byte(0x32);                                                    // 6 logIDs
    if (R.lid) {
        x.varint(R.lid_n);
        x.bytes(R.lid, R.lid_n);
    } else {
        const unsigned long long lid = a.first_log_id + R.line;
        x.varint(dma_dec_len(lid));
        x.dec(lid);
    }
    uint32_t sb;                                                     // 8 score
    memcpy(&sb, &a.scores[R.line], 4);
    x.byte(0x45);
    x.byte((uint8_t)sb); x.byte((uint8_t)(sb >> 8)); x.byte((uint8_t)(sb >> 16)); x.byte((uint8_t)(sb >> 24));
    x.byte(0x4A);                                                    // 9 extractedTimestamps (packed)
    x.varint(dma_varint_len((unsigned long long)R.ts));
    x.varint((unsigned long long)R.ts);
    x.bytes(F.pool + F.desc_off, F.desc_len);                        // 10 description
    x.byte(0x58);                                                    // 11 receivedTimestamp
    x.varint((unsigned long long)a.now);
    for (uint32_t j = 0; j < F.n_out; ++j) {                         // 12 alertsObtain, in key order
        if (R.pick[j] == DMA_NONE) continue;
        DmaOut t{nullptr, 0};
        dma_text(t, F, R, R.pick[j]);
        const uint32_t kl = F.out_len[j];
        x.byte(0x62);
        x.varint(1 + dma_varint_len(kl) + kl + 1 + dma_varint_len(t.n) + t.n);
        x.byte(0x0A);
        x.varint(kl);
        x.bytes(F.pool + F.out_off[j], kl);
        x.byte(0x12);
        x.varint(t.n);
        dma_text(x, F, R, R.pick[j]);
    }
}

// The alert keys a record's merged mask gives and the bit that supplies each (R.pick); returns the monitors whose values
// they need.
__device__ __forceinline__ unsigned long long dma_pick(const DmAlertFmt& F, uint32_t mask, DmaRec& R) {
    unsigned long long want = 0;
    for (uint32_t j = 0; j < F.n_out; ++j) {
        R.pick[j] = DMA_NONE;
        for (uint32_t t = F.sup_off[j]; t < F.sup_off[j + 1]; ++t)
            if (mask >> F.sup[t] & 1u) R.pick[j] = F.sup[t];
        if (R.pick[j] == DMA_NONE) continue;
        if (R.pick[j] < F.n_keys) want |= 1ull << R.pick[j];
        else
            for (uint32_t t = F.combo_off[R.pick[j] - F.n_keys]; t < F.combo_off[R.pick[j] - F.n_keys + 1]; ++t)
                want |= 1ull << F.members[t];
    }
    return want;
}

// Anomalous record r, its values and Time found: its varint-delimited DetectorSchema, written to w (or counted).
__device__ __forceinline__ void dma_finish(const DmAlertArgs& a, uint32_t r, const DmaRec& R, DmaOut& w) {
    DmaOut c{nullptr, 0};
    dma_body(c, a, R, r);
    w.varint(c.n);
    if (w.o) dma_body(w, a, R, r);
    else w.n += c.n;
}

// logIDs[0] of the record R.line: nothing to find for a raw line (R.lid = nullptr, the decimal number); for a LogSchema
// record the last `logID` (field 2, LEN) of its payload, "" when it has none, as protobuf reads it.  False where the
// payload does not walk (a record the unwrap kernels accepted always does).
__device__ __forceinline__ bool dma_log_id(const DmAlertArgs& a, DmaRec& R) {
    R.lid = nullptr;
    R.lid_n = 0;
    if (a.src != DMA_LOGS) return true;
    uint32_t pos = a.pay_off[R.line];
    const uint32_t end = pos + a.pay_len[R.line];
    R.lid = a.pay + pos;
    while (pos < end) {
        uint32_t field, wt;
        if (!dm_pb_tag(a.pay, pos, end, field, wt)) return false;
        if (wt != 2) {
            if (!dm_pb_skip(a.pay, pos, end, wt)) return false;
            continue;
        }
        uint64_t len;
        if (!dm_pb_varint(a.pay, pos, end, len) || len > (uint64_t)(end - pos)) return false;
        if (field == 2) { R.lid = a.pay + pos; R.lid_n = (uint32_t)len; }
        pos += (uint32_t)len;
    }
    return true;
}

// Anomalous record r of a key=value batch: its varint-delimited DetectorSchema, written to w (or counted).  False: the
// record declines.
__device__ bool dma_emit(const DmAlertArgs& a, uint32_t r, DmaOut& w) {
    const DmAlertFmt& F = *a.fmt;
    DmaRec R;
    R.line = a.rec_line[r];
    if (!dma_log_id(a, R)) return false;
    const unsigned long long off = a.rec_off[r];
    R.s = a.buf + off;
    R.ns = nullptr;
    uint32_t n = 0;
    while (off + n < a.nbytes && R.s[n] != 0x0Au) ++n;               // R-tok L1: the record ends at its '\n'
    const unsigned long long want = dma_pick(F, a.rec_mask[r], R) | 1ull << DMA_MSG;
    R.found = dma_fields(F, R.s, n, want, R.span);
    // extractedTimestamps (R-tok L7): the seconds of msg=audit(<Time>: or ), else the clock
    R.ts = a.now;
    if (R.found >> DMA_MSG & 1ull) {
        const uint8_t* v = R.s + R.span[DMA_MSG].b;
        const uint32_t vn = R.span[DMA_MSG].e - R.span[DMA_MSG].b;
        if (vn >= 6 && v[0] == 'a' && v[1] == 'u' && v[2] == 'd' && v[3] == 'i' && v[4] == 't' && v[5] == '(') {
            uint32_t j = 6;
            while (j < vn && v[j] != ':' && v[j] != ')') ++j;
            if (!dma_time(v + 6, j - 6, a.now, &R.ts)) return false;
        }
    }
    dma_finish(a, r, R, w);
    return true;
}

__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_size(DmAlertArgs a) {
    const uint32_t n = a.ahdr->n_alerts;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_entries; r += gridDim.x * blockDim.x) {
        unsigned long long bytes = 0;
        if (r < n) {
            DmaOut w{nullptr, 0};
            if (dma_emit(a, r, w)) bytes = w.n;
            else atomicOr(&a.ahdr->declined, 1u);
        }
        a.size[r] = bytes;
    }
}

__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_write(DmAlertArgs a) {
    const uint32_t n = a.ahdr->n_alerts;
    if (a.ahdr->declined || a.ahdr->total > a.out_cap) return;       // the host falls back; nothing is written
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        DmaOut w{a.out, a.size[r]};
        dma_emit(a, r, w);
    }
}

// ---------------------------------------------------------------------------------------------- log_format mode
// One thread per anomalous record, DM_FMTL_THREADS per CTA, the captures in dynamic shared memory as in
// dm_k_format_lanes: the header chain, (R-norm) the Content normalised again into nbuf at its own offset, the template
// chains, all through the matcher's device functions and in warp lockstep, then dm_fmtl_locate for every monitor.  The
// values are what the host's LogFormat.parse gives: header captures verbatim from the message, template variables as
// slices of the (normalised) Content.  Time is the header capture F.time_cap.  !WRITE: the size pass (and declines);
// WRITE: the write pass.
template <bool NORM, bool WRITE>
__global__ void __launch_bounds__(DM_FMTL_THREADS) dm_k_alert_format(DmAlertArgs a) {
#ifdef DM_EMU
    uint2* s_caps = reinterpret_cast<uint2*>(g_emu_dyn_smem.data());
#else
    extern __shared__ uint2 s_caps[];
#endif
    const DmFormat& f = *a.efmt;
    const DmAlertFmt& F = *a.fmt;
    const uint32_t n = a.ahdr->n_alerts;
    if (WRITE && (a.ahdr->declined || a.ahdr->total > a.out_cap)) return;
    const uint32_t tid = threadIdx.x;
    uint2* hcap = s_caps + tid;
    uint2* vcap = s_caps + f.max_slots * DM_FMTL_THREADS + tid;
    const uint32_t lim = WRITE ? n : a.n_entries;
    for (uint32_t wbase = blockIdx.x * blockDim.x + (tid & ~31u); wbase < lim; wbase += gridDim.x * blockDim.x) {
        const uint32_t r = wbase + (tid & 31u);
        const bool act = r < n;
        uint32_t s = 0, e = 0;
        if (act) {
            s = (uint32_t)a.rec_off[r];
            e = s;
            while (e < a.nbytes && a.buf[e] != 0x0Au) ++e;
        }
        const uint32_t n_hcaps = dm_fmtl_match_chain<true>(f, 0, a.buf, s, e, hcap, act);
        const bool hok = n_hcaps != 0xFFFFFFFFu;
        int32_t eid = -1;
        uint32_t n_vars = 0;
        if (f.content_capture != DM_FMT_NONE) {
            uint2 cc = make_uint2(0, 0);
            if (hok) cc = hcap[(uint32_t)__popc(f.chain_need[0] & ((1u << f.content_capture) - 1u)) * DM_FMTL_THREADS];
            if (NORM) {
                if (hok) cc.y = dm_fmtl_normalise(f, a.buf, a.nbuf, cc.x, cc.y);
                __syncwarp();
            }
            const uint8_t* tbuf = NORM ? a.nbuf : a.buf;
            for (uint32_t t = 1; t < f.n_chains; ++t) {
                const uint32_t nv = dm_fmtl_match_chain<!NORM>(f, t, tbuf, cc.x, cc.x + cc.y, vcap, hok && eid < 0);
                if (nv != 0xFFFFFFFFu) { eid = (int32_t)t - 1; n_vars = nv; }
            }
        }
        if (!act) {
            if (!WRITE && r < a.n_entries) a.size[r] = 0;
            continue;
        }
        DmaRec R;
        R.line = a.rec_line[r];
        R.s = a.buf;
        R.ns = a.nbuf;
        dma_pick(F, a.rec_mask[r], R);
        R.found = 0;
        for (uint32_t k = 0; k < F.n_keys; ++k) {
            uint2 cap;
            if (dm_fmtl_locate(f, k, hok, eid, n_hcaps, n_vars, hcap, vcap, cap)) {
                R.span[k].b = cap.x;
                R.span[k].e = cap.x + cap.y;
                R.span[k].nrm = (NORM && f.mon_source[k]) ? 1u : 0u;
                R.found |= 1ull << k;
            }
        }
        R.ts = a.now;
        bool ok = dma_log_id(a, R);
        if (ok && F.time_cap != DMA_NONE && hok && F.time_cap < n_hcaps) {
            const uint2 tc = hcap[(uint32_t)__popc(f.chain_need[0] & ((1u << F.time_cap) - 1u)) * DM_FMTL_THREADS];
            ok = dma_time(a.buf + tc.x, tc.y, a.now, &R.ts);
        }
        if (WRITE) {
            DmaOut w{a.out, a.size[r]};
            dma_finish(a, r, R, w);
        } else {
            unsigned long long bytes = 0;
            if (ok) {
                DmaOut w{nullptr, 0};
                dma_finish(a, r, R, w);
                bytes = w.n;
            } else {
                atomicOr(&a.ahdr->declined, 1u);
            }
            a.size[r] = bytes;
        }
    }
}

// ---------------------------------------------------------------------------------------------- ParserSchema batches
// One thread per anomalous record: the detection kernels' walk (dm_pb_walk_record_t) once more, now also keeping the
// logID and the Time entry.  Monitor k's value is what that walk found for it (a monitor is only flagged where the
// record has its value and, for an event monitor, its EventID); Time is logFormatVariables["Time"] as a str, absent =
// the clock.  !WRITE: the size pass (and declines); WRITE: the write pass.
template <bool WRITE>
__global__ void __launch_bounds__(DMA_THREADS) dm_k_alert_records(DmAlertArgs a) {
    __shared__ DmMonitors sm;
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(a.mons);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sm);
        for (uint32_t i = threadIdx.x; i < sizeof(DmMonitors) / 4; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const DmAlertFmt& F = *a.fmt;
    const uint32_t n = a.ahdr->n_alerts;
    if (WRITE && (a.ahdr->declined || a.ahdr->total > a.out_cap)) return;
    const uint32_t lim = WRITE ? n : a.n_entries;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < lim; r += gridDim.x * blockDim.x) {
        if (r >= n) { a.size[r] = 0; continue; }
        DmaRec R;
        R.line = a.rec_line[r];
        R.s = a.pay;
        R.ns = nullptr;
        const uint32_t pos = (uint32_t)a.rec_off[r];
        uint32_t vp[DM_MAX_KEYS], vl[DM_MAX_KEYS], present = 0;
        int32_t eid = 0;
        bool has_eid = false;
        DmPbMeta m;
        m.lid_p = pos; m.lid_l = 0; m.time_p = pos; m.time_l = 0; m.has_time = false;
        bool ok = dm_pb_walk_record_t<true>(a.pay, pos, pos + a.pay_len[R.line], sm, vp, vl, present, eid, has_eid, &m);
        dma_pick(F, a.rec_mask[r], R);
        R.found = 0;
        for (uint32_t k = 0; k < F.n_keys; ++k) {
            if (!(present >> k & 1u)) continue;
            R.span[k].b = vp[k];
            R.span[k].e = vp[k] + vl[k];
            R.span[k].nrm = 0;
            R.found |= 1ull << k;
        }
        R.lid = a.pay + m.lid_p;
        R.lid_n = m.lid_l;
        R.ts = a.now;
        if (ok && m.has_time) ok = dma_time(a.pay + m.time_p, m.time_l, a.now, &R.ts, true);
        if (WRITE) {
            DmaOut w{a.out, a.size[r]};
            dma_finish(a, r, R, w);
        } else {
            unsigned long long bytes = 0;
            if (ok) {
                DmaOut w{nullptr, 0};
                dma_finish(a, r, R, w);
                bytes = w.n;
            } else {
                atomicOr(&a.ahdr->declined, 1u);
            }
            a.size[r] = bytes;
        }
    }
}

// The matcher's format as the encoder needs it: the Time capture kept as well (chain_need), the slots recounted.
static inline void dm_alert_efmt_build(const DmFormat& f, uint32_t time_cap, DmFormat* out) {
    *out = f;
    if (time_cap < DM_FMT_MAX_CAPTURES) out->chain_need[0] |= 1u << time_cap;
    for (uint32_t c = 0; c < out->n_chains; ++c) {
        const uint32_t k = (uint32_t)__builtin_popcount(out->chain_need[c]);
        if (k > out->max_slots) out->max_slots = k;
    }
}

// ---------------------------------------------------------------------------------------------- host side
// Plain C++ from here on, shared by libdmdetect and the CPU emulator of tests/.
//
// The tiles of a scan over n elements.
static inline uint64_t dm_alert_tiles(uint64_t n) { return (n + DMA_TILE - 1) / DMA_TILE; }

// The encoder's scratch for max_lines records and an anomaly list of anomaly_cap entries, one block: per record + 1
// its rank (u32); per entry + 1 its offset and size (u64); the scans' tile sums (u64); per entry + 1 its record and
// merged mask (u32).  Carves the block at base into a's arrays and *tile_sums (base nullptr: only sizes it); returns
// its size in bytes.
static inline uint64_t dm_alert_scratch(uint8_t* base, uint64_t max_lines, uint32_t anomaly_cap, DmAlertArgs* a,
                                        unsigned long long** tile_sums) {
    const uint64_t lines = max_lines + 1, recs = (uint64_t)anomaly_cap + 1;
    const uint64_t off = (4 * lines + 7) & ~7ull, size = off + 8 * recs, tiles = size + 8 * recs;
    const uint64_t line = tiles + 8 * (dm_alert_tiles(lines > recs ? lines : recs) + 1), mask = line + 4 * recs;
    if (base) {
        a->rank = (uint32_t*)base;
        a->rec_off = (unsigned long long*)(base + off);
        a->size = (unsigned long long*)(base + size);
        *tile_sums = (unsigned long long*)(base + tiles);
        a->rec_line = (uint32_t*)(base + line);
        a->rec_mask = (uint32_t*)(base + mask);
    }
    return mask + 4 * recs;
}

// What the encoder takes from the last batch of source src (DMA_*): *n_lines records (ParserSchema: n_records, the
// others: the header's) and the anomaly entries it returns (ParserSchema: the flagged records, the others: the list's,
// at most its capacity).  0: nothing to word.  *declined: the batch declines before any launch, having more anomalous
// records than the per-record arrays hold (the return value is then their count).
static inline uint64_t dm_alert_entries(uint32_t src, const DmBatchHeader& hdr, uint64_t n_records, uint32_t anomaly_cap,
                                        uint64_t* n_lines, bool* declined) {
    const bool records = src == DMA_RECORDS;
    *n_lines = records ? n_records : hdr.n_lines;
    const uint64_t n = records ? hdr.n_anomalies : (hdr.anomaly_list_count < anomaly_cap ? hdr.anomaly_list_count : anomaly_cap);
    *declined = false;
    if (n == 0 || *n_lines == 0) return 0;
    *declined = n > anomaly_cap;
    return n;
}

// The instantiations the encoder runs.
typedef void (*DmAlertKernel)(DmAlertArgs);

// Marking the anomalous records (!gather) and gathering their masks: one thread per anomaly entry, or for ParserSchema
// batches one per record (*items: what the threads stride over).
static inline DmAlertKernel dm_alert_mark_kernel(uint32_t src, bool gather, uint64_t n_lines, uint64_t entries,
                                                 uint64_t* items) {
    *items = src == DMA_RECORDS ? n_lines : entries;
    if (src == DMA_RECORDS) return gather ? dm_k_alert_gather_records : dm_k_alert_mark_records;
    return gather ? dm_k_alert_gather : dm_k_alert_mark;
}

// The size (!write) and the write pass, one thread per anomalous record.  fmt: the batch was detected in log_format
// mode, norm: with R-norm.  *fmtl: the pass is dm_k_alert_format, which runs DM_FMTL_THREADS per CTA with the
// captures in dynamic shared memory (the others run DMA_THREADS per CTA).
static inline DmAlertKernel dm_alert_pass_kernel(uint32_t src, bool fmt, bool norm, bool write, bool* fmtl) {
    *fmtl = src != DMA_RECORDS && fmt;
    if (src == DMA_RECORDS) return write ? dm_k_alert_records<true> : dm_k_alert_records<false>;
    if (!fmt) return write ? dm_k_alert_write : dm_k_alert_size;
    if (norm) return write ? dm_k_alert_format<true, true> : dm_k_alert_format<true, false>;
    return write ? dm_k_alert_format<false, true> : dm_k_alert_format<false, false>;
}

// Fills f from the handle's keys and dm_set_alert_format's arguments.  strings = version, detectorID, detectorType,
// description, then the n_strings - 4 alert keys in output order; alert key j is supplied by the mask bits
// bits[bits_off[j], bits_off[j + 1]).  Returns nullptr or the reason the arguments are refused.
static inline const char* dm_alert_fmt_build(const DmKeys& keys, uint32_t n_strings, const uint8_t* blob,
                                             const uint32_t* lens, const uint32_t* bits_off, const uint32_t* bits,
                                             uint32_t n_combos, const uint32_t* combo_off, const uint32_t* members,
                                             uint32_t time_cap, DmAlertFmt* f) {
    memset(f, 0, sizeof(*f));
    if (n_strings < 4) return "at least 4 strings: version, detectorID, detectorType, description";
    const uint32_t n_out = n_strings - 4;
    if (n_out > DM_MAX_KEYS) return "more than 32 alert keys";
    if (keys.n + n_combos > DM_MAX_KEYS) return "monitors + combinations exceed the 32 mask bits";
    if (n_out && (!bits_off || !bits || bits_off[0] != 0)) return "bits_off must start at 0";
    for (uint32_t j = 0; j < n_out; ++j) {
        if (bits_off[j + 1] < bits_off[j] || bits_off[j + 1] > DM_MAX_KEYS) return "bits_off is not increasing or holds more than 32 bits";
        for (uint32_t t = bits_off[j]; t < bits_off[j + 1]; ++t)
            if (bits[t] >= keys.n + n_combos) return "a supplying bit is neither a monitor nor a combination";
    }
    if (n_combos && (!combo_off || !members || combo_off[0] != 0)) return "combo_off must start at 0";
    if (n_combos && combo_off[n_combos] > DM_MAX_COMBO_MEMBERS) return "more than 64 combination members";
    for (uint32_t c = 0; c < n_combos; ++c) {
        if (combo_off[c + 1] <= combo_off[c]) return "a combination is empty or combo_off is not increasing";
        for (uint32_t t = combo_off[c]; t < combo_off[c + 1]; ++t)
            if (members[t] >= keys.n) return "a combination member is not a monitor";
    }
    f->n_keys = keys.n;
    f->n_out = n_out;
    f->time_cap = time_cap < DM_FMT_MAX_CAPTURES ? time_cap : DMA_NONE;
    for (uint32_t k = 0; k < keys.n; ++k) {
        f->key_len[k] = keys.len[k];
        memcpy(f->key[k], keys.bytes[k], keys.len[k]);
    }
    f->key_len[DMA_MSG] = 3;
    memcpy(f->key[DMA_MSG], "msg", 3);
    for (uint32_t j = 0; j <= n_out; ++j) f->sup_off[j] = n_out ? bits_off[j] : 0;
    for (uint32_t t = 0; n_out && t < bits_off[n_out]; ++t) f->sup[t] = (uint8_t)bits[t];
    f->n_combos = n_combos;
    for (uint32_t c = 0; n_combos && c <= n_combos; ++c) f->combo_off[c] = combo_off[c];
    for (uint32_t t = 0; n_combos && t < combo_off[n_combos]; ++t) f->members[t] = (uint8_t)members[t];
    // the pool: fields 1-3 and 10 with their tags and lengths, then the alert keys
    uint64_t pos = 0, src = 0;
    auto put = [&](const uint8_t* p, uint64_t n) -> bool {
        if (pos + n > DMA_POOL) return false;
        memcpy(f->pool + pos, p, n);
        pos += n;
        return true;
    };
    auto field = [&](uint8_t tag, const uint8_t* p, uint64_t n) -> bool {
        uint8_t hdr[11];
        int k = 0;
        hdr[k++] = tag;
        uint64_t v = n;
        while (v >= 0x80u) { hdr[k++] = (uint8_t)(v | 0x80u); v >>= 7; }
        hdr[k++] = (uint8_t)v;
        return put(hdr, k) && put(p, n);
    };
    const uint8_t tags[4] = {0x0A, 0x12, 0x1A, 0x52};
    for (uint32_t i = 0; i < 4; ++i) {
        if (i == 3) f->desc_off = (uint32_t)pos;
        if (!field(tags[i], blob + src, lens[i])) return "the strings exceed 16 KiB";
        src += lens[i];
        if (i == 2) f->head_len = (uint32_t)pos;
    }
    f->desc_len = (uint32_t)pos - f->desc_off;
    for (uint32_t j = 0; j < n_out; ++j) {
        f->out_off[j] = (uint32_t)pos;
        f->out_len[j] = lens[4 + j];
        if (!put(blob + src, lens[4 + j])) return "the strings exceed 16 KiB";
        src += lens[4 + j];
    }
    return nullptr;
}
