// dm_kernels_logs.cuh -- LogSchema input: the reader stage's records (one serialized LogSchema per message, or a
// varint-length-delimited batch of them) unwrapped on the device into the '\n'-terminated text the line kernels take.
//
//   LogSchema   1 __version__   2 logID   3 log   4 logSource   5 hostname      (all proto3 strings)
//
// Rule R-log (DESIGN.md): a record is well-formed exactly when protobuf's runtime parses it as LogSchema, except that
// a group makes it malformed (dm_pb.cuh, as for ParserSchema); strict UTF-8 in fields 1-5.  Its text is the last `log`
// field ("" when absent) less ONE trailing '\n'; a text that still holds a '\n' is unusable.  Malformed and unusable
// records get flag and score 0, count as bad_records and take no training slot.  Every other record gets the result its
// text gets as one line of a raw-line message made of the usable texts, in order.
//
// Four launches before the line path, one after it:
//   dm_k_logs_walk     one thread per record: field walk, text bounds, and the exclusive scan of (text + '\n' bytes,
//                      usable) inside the CTA's chunk of records
//   dm_k_logs_scan     one CTA: exclusive scan of the chunk totals; totals into the DmLogsHeader the host reads back
//   dm_k_logs_compact  one thread per record: the record <-> line maps and the offsets of each line
//   dm_k_logs_copy     one thread per 16 OUTPUT bytes: the compacted texts with one 16-byte store each, so that one
//                      8 MiB record is copied by the whole grid and not by one thread; then the zeroed slack
//   (the line path of dm_process_lines on the compacted buffer)
//   dm_k_logs_scatter  flags / scores back to record order, anomaly entries to (record, mask, payload offset in the
//                      caller's message), statistics corrected from the compacted message to the caller's
#pragma once
#include "dm_device.cuh"
#include "dm_pb.cuh"

#define DML_THREADS 256
#define DML_UNUSABLE 0xFFFFFFFFu
#define DML_SLACK 64u                      // zeroed bytes after the compacted texts (what the line kernels read past)

// Written by the unwrap kernels; the host reads it back with one copy.
struct DmLogsHeader {
    unsigned long long total_bytes;        // compacted bytes: every usable text plus its '\n'
    unsigned long long n_lines;            // usable records
    unsigned long long n_train;            // min(n_train_records, n_lines): the records that train
    unsigned long long bound;              // first record scored: just past the n_train_records-th usable one, n_records
                                           // when there are fewer, 0 when n_train_records is 0
};

struct DmLogsArgs {
    const uint8_t* buf;                    // the caller's message
    const uint32_t* rec_off;               // per record: offset of its payload (after the length prefix)
    const uint32_t* rec_len;               // per record: payload length
    uint32_t n_records;
    uint32_t n_train_records;
    uint32_t per_cta;                      // records per chunk of dm_k_logs_walk (a multiple of DML_THREADS)
    uint32_t n_chunks;
    uint32_t* text_off;                    // per record: offset of its text in buf
    uint32_t* text_len;                    // per record: text length without the dropped '\n'; DML_UNUSABLE if none
    unsigned long long* loc;               // per record: exclusive prefix in its chunk, bytes | lines << 32
    unsigned long long* chunk;             // per chunk: its total, then (dm_k_logs_scan) the prefix in front of it
    uint32_t* rec_line;                    // per record: its line in the compacted buffer, DML_UNUSABLE if none
    uint32_t* line_src;                    // per line: offset of its text in buf
    uint32_t* line_dst;                    // per line: offset of its text in out; [n_lines] = total_bytes
    uint32_t* line_rec;                    // per line: its record
    uint8_t* out;                          // the compacted buffer (16-byte aligned)
    uint64_t out_cap;                      // bytes of out (a multiple of 16)
    DmLogsHeader* lhdr;
};

// Walks one LogSchema record [pos, end).  False where protobuf's runtime refuses the record, and for a group; else
// [tp, tp + tl) is the last `log` field (tl = 0 when there is none).  A field 1-5 under another wire type is an
// unknown field to protobuf and skipped; an unknown LEN field is not checked for UTF-8.
__device__ __forceinline__ bool dm_pb_walk_log(const uint8_t* __restrict__ buf, uint32_t pos, const uint32_t end,
                                               uint32_t& tp, uint32_t& tl) {
    tp = pos;
    tl = 0;
    while (pos < end) {
        uint32_t field, wt;
        if (!dm_pb_tag(buf, pos, end, field, wt)) return false;
        if (wt != 2) {
            if (!dm_pb_skip(buf, pos, end, wt)) return false;
            continue;
        }
        uint64_t len64;
        if (!dm_pb_varint(buf, pos, end, len64) || len64 > (uint64_t)(end - pos)) return false;
        const uint32_t len = (uint32_t)len64;
        if (field <= 5u && !dm_utf8_ok(buf + pos, len)) return false;
        if (field == 3u) { tp = pos; tl = len; }
        pos += len;
    }
    return true;
}

// Exclusive scan of v over the CTA (every thread calls it); total = the CTA's sum.
__device__ __forceinline__ unsigned long long dml_cta_scan(unsigned long long v, unsigned long long* s_warp,
                                                           unsigned long long& total) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (uint32_t d = 1; d < 32u; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31u) s_warp[warp] = x;
    __syncthreads();
    unsigned long long before = 0, all = 0;
#pragma unroll
    for (uint32_t w = 0; w < DML_THREADS / 32; ++w) {
        const unsigned long long s = s_warp[w];
        before += w < warp ? s : 0ull;
        all += s;
    }
    __syncthreads();
    total = all;
    return before + x - v;
}

// CTA b owns records [b * per_cta, (b + 1) * per_cta) and walks them DML_THREADS at a time.  A usable record adds
// (text length + 1) bytes and one line; both are scanned as one 64-bit word (bytes below 2^32: they never exceed the
// message, which is below 2^32).
__global__ void __launch_bounds__(DML_THREADS) dm_k_logs_walk(DmLogsArgs a) {
    __shared__ unsigned long long s_warp[DML_THREADS / 32];
    const uint8_t* __restrict__ buf = a.buf;
    const uint32_t lo = blockIdx.x * a.per_cta;
    const uint32_t hi = a.n_records - lo < a.per_cta ? a.n_records : lo + a.per_cta;
    unsigned long long carry = 0;
    for (uint32_t base = lo; base < hi; base += DML_THREADS) {
        const uint32_t r = base + threadIdx.x;
        unsigned long long v = 0;
        if (r < hi) {
            const uint32_t p = a.rec_off[r];
            uint32_t tp, tl;
            bool ok = dm_pb_walk_log(buf, p, p + a.rec_len[r], tp, tl);
            if (ok && tl && buf[tp + tl - 1] == 0x0Au) --tl;                 // one trailing '\n' is dropped
            for (uint32_t i = 0; ok && i < tl; ++i)
                if (buf[tp + i] == 0x0Au) ok = false;                         // a text of two lines is unusable
            a.text_off[r] = tp;
            a.text_len[r] = ok ? tl : DML_UNUSABLE;
            if (ok) v = (1ull << 32) | (unsigned long long)(tl + 1u);
        }
        unsigned long long tot;
        const unsigned long long ex = dml_cta_scan(v, s_warp, tot);
        if (r < hi) a.loc[r] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) a.chunk[blockIdx.x] = carry;
}

// One CTA: the chunk totals become the prefix in front of each chunk; the batch totals go to the header.
__global__ void __launch_bounds__(DML_THREADS) dm_k_logs_scan(DmLogsArgs a) {
    __shared__ unsigned long long s_warp[DML_THREADS / 32];
    unsigned long long carry = 0;
    for (uint32_t base = 0; base < a.n_chunks; base += DML_THREADS) {
        const uint32_t c = base + threadIdx.x;
        const unsigned long long v = c < a.n_chunks ? a.chunk[c] : 0ull;
        unsigned long long tot;
        const unsigned long long ex = dml_cta_scan(v, s_warp, tot);
        if (c < a.n_chunks) a.chunk[c] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) {
        const unsigned long long lines = carry >> 32, bytes = carry & 0xFFFFFFFFull;
        a.lhdr->total_bytes = bytes;
        a.lhdr->n_lines = lines;
        a.lhdr->n_train = a.n_train_records < lines ? a.n_train_records : lines;
        // the split as dm_k_records_bound puts it: past the n_train_records-th usable record (dm_k_logs_compact), the
        // whole batch when it holds fewer
        a.lhdr->bound = a.n_train_records > lines ? a.n_records : 0ull;
        a.line_dst[lines] = (uint32_t)bytes;
    }
}

__global__ void __launch_bounds__(DML_THREADS) dm_k_logs_compact(DmLogsArgs a) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_records; r += gridDim.x * blockDim.x) {
        if (a.text_len[r] == DML_UNUSABLE) { a.rec_line[r] = DML_UNUSABLE; continue; }
        const unsigned long long p = a.chunk[r / a.per_cta] + a.loc[r];
        const uint32_t u = (uint32_t)(p >> 32);
        a.rec_line[r] = u;
        a.line_src[u] = a.text_off[r];
        a.line_dst[u] = (uint32_t)p;
        a.line_rec[u] = r;
        if (u + 1ull == a.n_train_records) a.lhdr->bound = r + 1ull;
    }
}

// Thread t writes out[16t, 16t + 16): a binary search over line_dst finds the line of its first byte, later bytes step
// to the next line where one ends (every line holds at least its '\n').  Bytes from total_bytes to the end of the
// slack are zero.  The grid is sized from the message length before the total is known; threads past it store nothing.
__global__ void __launch_bounds__(DML_THREADS) dm_k_logs_copy(DmLogsArgs a) {
    const uint8_t* __restrict__ buf = a.buf;
    const uint64_t total = a.lhdr->total_bytes;
    const uint32_t n_lines = (uint32_t)a.lhdr->n_lines;
    uint64_t end = (total + DML_SLACK + 15u) & ~15ull;
    if (end > a.out_cap) end = a.out_cap;
    const uint64_t step = 16ull * gridDim.x * blockDim.x;
    for (uint64_t o = 16ull * (blockIdx.x * blockDim.x + threadIdx.x); o < end; o += step) {
        uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
        if (o < total) {
            uint32_t lo = 0, hi = n_lines - 1;                                // the last line starting at or before o
            while (lo < hi) {
                const uint32_t mid = (lo + hi + 1u) >> 1;
                if (a.line_dst[mid] <= o) lo = mid; else hi = mid - 1u;
            }
            uint32_t u = lo;
            uint64_t ls = a.line_dst[u], le = a.line_dst[u + 1];              // [ls, le) = text + '\n'
            const uint8_t* src = buf + a.line_src[u];
#pragma unroll
            for (uint32_t i = 0; i < 16u; ++i) {
                const uint64_t p = o + i;
                uint32_t b = 0;
                if (p < total) {
                    while (p >= le) { ++u; ls = le; le = a.line_dst[u + 1]; src = buf + a.line_src[u]; }
                    b = p + 1 == le ? 0x0Au : (uint32_t)src[p - ls];
                }
                const uint32_t sh = 8u * (i & 3u);
                if (i < 4) w0 |= b << sh; else if (i < 8) w1 |= b << sh; else if (i < 12) w2 |= b << sh; else w3 |= b << sh;
            }
        }
        *reinterpret_cast<uint4*>(a.out + o) = make_uint4(w0, w1, w2, w3);
    }
}

// After the line path: per-record outputs, the anomaly list rewritten in place, the statistics corrected.  The line
// path counted n_lines records of total_bytes bytes, n_train of them trained; the message holds n_records records of
// nbytes bytes, the malformed and unusable ones are bad_records, and detect_lines counts every record from the bound on
// (as for ParserSchema batches).
__global__ void __launch_bounds__(DML_THREADS) dm_k_logs_scatter(DmLogsArgs a, const uint8_t* __restrict__ line_flags,
                                                                 const float* __restrict__ line_scores, uint8_t* flags,
                                                                 float* scores, dm_anomaly_t* anoms, uint32_t anomaly_cap,
                                                                 DmBatchHeader* hdr, unsigned long long* stats, uint64_t nbytes) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    for (uint32_t r = tid; r < a.n_records; r += nth) {
        const uint32_t u = a.rec_line[r];
        flags[r] = u == DML_UNUSABLE ? 0 : line_flags[u];
        scores[r] = u == DML_UNUSABLE ? 0.0f : line_scores[u];
    }
    const uint32_t n_list = hdr->anomaly_list_count < anomaly_cap ? hdr->anomaly_list_count : anomaly_cap;
    for (uint32_t i = tid; i < n_list; i += nth) {
        const uint32_t r = a.line_rec[anoms[i].line];
        anoms[i].line = r;
        anoms[i].offset = a.rec_off[r];
    }
    if (tid == 0) {
        const DmLogsHeader h = *a.lhdr;
        const unsigned long long n = a.n_records, bad = n - h.n_lines;
        stats[0] += bad;
        stats[2] += (n - h.bound) - (h.n_lines - h.n_train);
        stats[5] += nbytes - h.total_bytes;                                  // (mod 2^64: a bare empty record compacts to 1 byte)
        stats[7] += bad;
        hdr->n_lines = n;
    }
}
