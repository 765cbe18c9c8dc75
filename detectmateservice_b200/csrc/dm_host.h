// dm_host.h -- host steps of a call that feed no single kernel: the framing of a varint-length-delimited message, the
// merge of a batch's anomaly entries and the statistics a synchronous record call counts on the host.  Plain C++ (no
// CUDA runtime calls): shared by libdmdetect and the CPU emulator harness of tests/.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/dmdetect.h"

#define DM_FRAME_TRUNCATED 1      // a length prefix ends with the message, or runs past 10 bytes
#define DM_FRAME_PAST_END 2       // a record runs past the end of the message

// varint length, payload, varint length, payload ... split into the payloads.  On an error, `error` is one of
// DM_FRAME_*, `at` the byte it was found at and, for DM_FRAME_PAST_END, `rec_len` the length the prefix gave.
struct DmFrames {
    std::vector<uint32_t> off, len;
    int error = 0;
    uint64_t at = 0, rec_len = 0;
};

inline DmFrames dm_frame_split(const uint8_t* buf, uint64_t nbytes) {
    DmFrames f;
    uint64_t pos = 0;
    while (pos < nbytes) {
        uint64_t l = 0;
        int shift = 0;
        for (;;) {
            if (pos >= nbytes || shift > 63) { f.error = DM_FRAME_TRUNCATED; f.at = pos; return f; }
            const uint8_t b = buf[pos++];
            l |= (uint64_t)(b & 0x7F) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (l > nbytes - pos) { f.error = DM_FRAME_PAST_END; f.at = pos; f.rec_len = l; return f; }
        f.off.push_back((uint32_t)pos);
        f.len.push_back((uint32_t)l);
        pos += l;
    }
    return f;
}

// The records of a LogSchema message: the payloads of a delimited batch, or the whole message as one bare record.
inline DmFrames dm_frame_records(const uint8_t* buf, uint64_t nbytes, bool delimited) {
    if (delimited) return dm_frame_split(buf, nbytes);
    DmFrames f;
    f.off.push_back(0);
    f.len.push_back((uint32_t)nbytes);
    return f;
}

// A buffer that must hold `need` bytes and holds `cap`: the capacity to grow it to, or `cap` when it is large enough.
// Grows at least twofold, so that a stream of slowly growing messages reallocates a logarithmic number of times.
inline uint64_t dm_grow_cap(uint64_t cap, uint64_t need) {
    if (need <= cap) return cap;
    return std::max<uint64_t>(need, std::max<uint64_t>(2 * cap, 1u << 20));
}

// The kernels append one anomaly entry per unknown field: sorts the n entries by record and merges those of one record
// (mask = the OR of theirs).  Returns the number of records.
inline uint32_t dm_anomalies_merge(dm_anomaly_t* v, uint32_t n) {
    std::sort(v, v + n, [](const dm_anomaly_t& a, const dm_anomaly_t& b) { return a.line < b.line; });
    uint32_t m = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (m && v[m - 1].line == v[i].line) { v[m - 1].mask |= v[i].mask; continue; }
        v[m++] = v[i];
    }
    return m;
}

// The keys a window with keys carries: novel-list entries [from, to) of the `learnt` keys this rank has learnt so far
// (at most novel_cap are listed), of which `exported` have travelled already; at most `cap` per window, the rest
// (`pending`) waits for the next window.  Truncating instead of failing keeps every rank in the collective.
struct DmWindowKeys { uint64_t from, to, pending; };
inline DmWindowKeys dm_window_keys(uint64_t exported, uint64_t learnt, uint64_t novel_cap, uint64_t cap) {
    const uint64_t listed = std::min(learnt, novel_cap);
    const uint64_t to = std::min(listed, exported + cap);
    return DmWindowKeys{exported, to, listed - to};
}

// What a synchronous record call (dm_process_values, dm_process_records) adds to the statistics words on the host:
// lines, train_lines, detect_lines and bytes.
inline void dm_stats_add_records(unsigned long long* w, uint64_t n_records, uint64_t trained, uint64_t scored, uint64_t nbytes) {
    w[0] += n_records;
    w[1] += trained;
    w[2] += scored;
    w[5] += nbytes;
}
