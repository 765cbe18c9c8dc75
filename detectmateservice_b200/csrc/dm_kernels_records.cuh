// dm_kernels_records.cuh -- record mode on the GPU: a batch of serialized ParserSchema
// records (the reference's real wire format of the detector's input,
// /root/reference/container/fluentout/schemas_pb.rb:8; one record per NNG message today,
// engine.py:163-187) walked, matched against the configured monitors, hashed and probed on
// the device.  One thread per record.
//
//   ParserSchema   4 EventID int32 (varint)            6 variables repeated string
//                 10 logFormatVariables map<string,string> (entry: 1 key, 2 value)
//   every other field is skipped by wire type.
//
// Well-formed (DESIGN.md section 5.3): a record is walked exactly as protobuf's runtime parses ParserSchema -- tags of
// at most 5 bytes below 2^32 and not field 0, every fixed32/fixed64/LEN payload inside the record, strict UTF-8 in the
// string fields and in map keys and values -- except that a group (wire types 3/4) makes the record malformed.  A
// malformed record has flag, score and mask 0, is counted in stats word 7 (bad_records) and never trains.
//
// Monitor semantics (R-spec 3, DESIGN.md): a global monitor applies to every record, an
// event monitor only when record.EventID matches; header monitors read
// logFormatVariables[KEY] (last entry wins, as in protobuf maps), variable monitors read
// variables[i]; a missing field skips the monitor.
#pragma once
#include "dm_device.cuh"

struct DmMonitor {
    int32_t event_id;
    uint32_t has_event;      // 0 = global scope
    uint32_t source;         // 0 = header variable (by key), 1 = variable (by index)
    uint32_t var_index;
    uint32_t key_len;
    uint8_t key[64];
};

// Combination monitors (NewValueComboDetector, DESIGN.md R-combo): combo c is the ordered
// tuple of the values of monitors combo_members[combo_off[c] .. combo_off[c+1]); its table
// field (salt) and output-mask bit are n + c.  A monitor whose member_only bit is set does
// not alert on its own.
#define DM_MAX_COMBO_MEMBERS 64
struct DmMonitors {
    uint32_t n;
    uint32_t n_combos;
    uint32_t member_only;
    uint32_t pad_;
    uint32_t combo_off[DM_MAX_KEYS + 1];
    uint8_t combo_members[DM_MAX_COMBO_MEMBERS];
    uint32_t pad2_[3];
    DmMonitor m[DM_MAX_KEYS];
};

// Fingerprint of an ordered tuple of value fingerprints (order-sensitive fold).
DM_HD uint64_t dm_combo_fold(uint64_t acc, uint64_t fp) { return dm_splitmix64(acc ^ fp); }
DM_HD uint64_t dm_combo_seed(uint32_t n_members) { return 0xC0B0C0B0ull + 0x9E3779B97F4A7C15ull * (uint64_t)n_members; }

struct DmRecordsArgs {
    const uint8_t* buf;
    const uint32_t* rec_off;       // n_records + 1 offsets of the record payloads (after the length prefix)
    const uint32_t* rec_len;       // payload lengths
    uint32_t n_records;
    uint32_t n_train_records;
    const DmMonitors* mons;
    DmTable table;
    uint8_t* flags;
    float* scores;
    uint32_t* masks;
    DmBatchHeader* hdr;
    unsigned long long* stats;
};

__device__ __forceinline__ bool dm_pb_varint(const uint8_t* __restrict__ buf, uint32_t& pos, uint32_t end, uint64_t& out) {
    uint64_t v = 0;
    for (uint32_t shift = 0; shift < 70; shift += 7) {
        if (pos >= end) return false;
        const uint32_t b = buf[pos++];
        v |= (uint64_t)(b & 0x7Fu) << shift;
        if (!(b & 0x80u)) { out = v; return true; }
    }
    return false;
}

// A tag as protobuf's runtime reads it: at most 5 bytes, below 2^32, field number not 0.
__device__ __forceinline__ bool dm_pb_tag(const uint8_t* __restrict__ buf, uint32_t& pos, uint32_t end, uint32_t& field, uint32_t& wt) {
    uint64_t v = 0;
    for (uint32_t shift = 0; shift < 35; shift += 7) {
        if (pos >= end) return false;
        const uint32_t b = buf[pos++];
        v |= (uint64_t)(b & 0x7Fu) << shift;
        if (!(b & 0x80u)) {
            field = (uint32_t)(v >> 3);
            wt = (uint32_t)v & 7u;
            return (v >> 32) == 0 && field != 0;
        }
    }
    return false;
}

// Skips the payload of a field protobuf does not know (or knows under another wire type).  Groups (wire types 3/4)
// are refused: proto3 cannot declare them, so no ParserSchema producer emits them -- the one deliberate divergence
// from protobuf's runtime, which skips a group as an unknown field.
__device__ __forceinline__ bool dm_pb_skip(const uint8_t* __restrict__ buf, uint32_t& pos, uint32_t end, uint32_t wt) {
    uint64_t v;
    switch (wt) {
        case 0: return dm_pb_varint(buf, pos, end, v);
        case 1: if (end - pos < 8u) return false; pos += 8; return true;
        case 5: if (end - pos < 4u) return false; pos += 4; return true;
        case 2:
            if (!dm_pb_varint(buf, pos, end, v) || v > (uint64_t)(end - pos)) return false;
            pos += (uint32_t)v;
            return true;
        default: return false;
    }
}

// Strict UTF-8 (what protobuf's runtime checks in every proto3 string): no overlong forms, no surrogates, nothing
// above U+10FFFF, no sequence cut short.
__device__ __forceinline__ bool dm_utf8_ok(const uint8_t* __restrict__ s, uint32_t n) {
    uint32_t i = 0;
    while (i < n) {
        const uint32_t c = s[i];
        if (c < 0x80u) { ++i; continue; }
        uint32_t need, lo = 0x80u, hi = 0xBFu;
        if (c >= 0xC2u && c <= 0xDFu) need = 1;
        else if (c >= 0xE0u && c <= 0xEFu) { need = 2; if (c == 0xE0u) lo = 0xA0u; else if (c == 0xEDu) hi = 0x9Fu; }
        else if (c >= 0xF0u && c <= 0xF4u) { need = 3; if (c == 0xF0u) lo = 0x90u; else if (c == 0xF4u) hi = 0x8Fu; }
        else return false;
        if (n - i <= need) return false;
        const uint32_t c1 = s[i + 1];
        if (c1 < lo || c1 > hi) return false;
        for (uint32_t j = 2; j <= need; ++j)
            if ((s[i + j] & 0xC0u) != 0x80u) return false;
        i += need + 1;
    }
    return true;
}

// The string fields of ParserSchema (1 2 3 5 6 7 8 9; 10 is the map, its keys and values are strings too).
DM_HD bool dm_pb_string_field(uint32_t f) { return f <= 9u && ((0x3EEu >> f) & 1u); }

// Walks one ParserSchema record [pos, end).  Returns false exactly where protobuf's runtime refuses the record (and for
// a group anywhere in it); else vp/vl/present hold the monitored values and eid/has_eid the EventID, as protobuf reads
// them: the last EventID wins, variables[i] is the i-th field 6, logFormatVariables[key] the last entry with that key.
// A map entry holding anything but LEN fields 1 and 2 is dropped, as protobuf's runtime drops it (its key and value are
// still checked for UTF-8); an absent key or value reads as "".
__device__ __forceinline__ bool dm_pb_walk_record(const uint8_t* __restrict__ buf, uint32_t pos, const uint32_t end,
                                                  const DmMonitors& sm, uint32_t* vp, uint32_t* vl, uint32_t& present,
                                                  int32_t& eid, bool& has_eid) {
    uint32_t var_idx = 0;
    while (pos < end) {
        uint32_t field, wt;
        if (!dm_pb_tag(buf, pos, end, field, wt)) return false;
        if (wt == 0 && field == 4) {
            uint64_t v;
            if (!dm_pb_varint(buf, pos, end, v)) return false;
            eid = (int32_t)(uint32_t)v;
            has_eid = true;
            continue;
        }
        if (wt != 2) {
            if (!dm_pb_skip(buf, pos, end, wt)) return false;
            continue;
        }
        uint64_t len64;
        if (!dm_pb_varint(buf, pos, end, len64) || len64 > (uint64_t)(end - pos)) return false;
        const uint32_t len = (uint32_t)len64;
        if (dm_pb_string_field(field) && !dm_utf8_ok(buf + pos, len)) return false;
        if (field == 6) {
            for (uint32_t k = 0; k < sm.n; ++k)
                if (sm.m[k].source == 1 && sm.m[k].var_index == var_idx) { vp[k] = pos; vl[k] = len; present |= 1u << k; }
            ++var_idx;
        } else if (field == 10) {
            uint32_t p = pos, kp = pos, kl = 0, xp = pos, xl = 0;      // key, value (absent = empty)
            const uint32_t e = pos + len;
            bool foreign = false;
            while (p < e) {
                uint32_t f2, w2;
                if (!dm_pb_tag(buf, p, e, f2, w2)) return false;
                if (w2 != 2 || (f2 != 1 && f2 != 2)) {
                    if (!dm_pb_skip(buf, p, e, w2)) return false;
                    foreign = true;
                    continue;
                }
                uint64_t l2;
                if (!dm_pb_varint(buf, p, e, l2) || l2 > (uint64_t)(e - p)) return false;
                if (!dm_utf8_ok(buf + p, (uint32_t)l2)) return false;
                if (f2 == 1) { kp = p; kl = (uint32_t)l2; }
                else { xp = p; xl = (uint32_t)l2; }
                p += (uint32_t)l2;
            }
            if (!foreign) {
                for (uint32_t k = 0; k < sm.n; ++k) {
                    if (sm.m[k].source != 0 || sm.m[k].key_len != kl) continue;
                    bool eq = true;
                    for (uint32_t i = 0; i < kl; ++i)
                        if (buf[kp + i] != sm.m[k].key[i]) { eq = false; break; }
                    if (eq) { vp[k] = xp; vl[k] = xl; present |= 1u << k; }
                }
            }
        }
        pos += len;
    }
    return true;
}

// phase 2: mark each record well-formed (flags[r] = 1) or not, for dm_k_records_bound;
// phase 0: the records before the split insert (training); phase 1: the others are scored (separate launches so that
// detection sees every insert).  Every record writes its outputs in phase 0 or 1.
// bound: {first scored record, records trained} from dm_k_records_bound, which puts the split just past the
// n_train_records-th WELL-FORMED record; NULL splits at record n_train_records itself (the same when it is 0).
__global__ void __launch_bounds__(128) dm_k_records(DmRecordsArgs a, int phase, const uint32_t* bound_in = nullptr) {
    __shared__ DmMonitors sm;
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(a.mons);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sm);
        for (uint32_t i = threadIdx.x; i < sizeof(DmMonitors) / 4; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const uint8_t* __restrict__ buf = a.buf;
    const uint32_t bound = bound_in ? bound_in[0] : a.n_train_records;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_records; r += gridDim.x * blockDim.x) {
        const bool train = r < bound;
        if (phase != 2 && train != (phase == 0)) continue;
        uint32_t vp[DM_MAX_KEYS], vl[DM_MAX_KEYS];
        uint32_t present = 0;
        int32_t eid = 0;
        bool has_eid = false;
        const uint32_t pos = a.rec_off[r];
        const bool ok = dm_pb_walk_record(buf, pos, pos + a.rec_len[r], sm, vp, vl, present, eid, has_eid);
        if (phase == 2) { a.flags[r] = ok ? 1 : 0; continue; }
        if (!ok) {                                                // malformed record: counted, never trained or scored
            a.flags[r] = 0; a.scores[r] = 0.0f; a.masks[r] = 0;
            atomicAdd(a.stats + 7, 1ull);
            continue;
        }
        uint32_t unknown = 0, have = 0;
        uint64_t fpv[DM_MAX_KEYS];
        for (uint32_t k = 0; k < sm.n; ++k) {
            if (!((present >> k) & 1u)) continue;
            if (sm.m[k].has_event && !(has_eid && eid == sm.m[k].event_id)) continue;
            const uint64_t fp = dm_fp64_bytes(buf + vp[k], vl[k]);
            fpv[k] = fp;
            have |= 1u << k;
            if ((sm.member_only >> k) & 1u) continue;
            const uint64_t key = dm_make_key(fp, dm_field_salt(k));
            if (train) dm_table_insert(a.table, key, &a.hdr->error);
            else if (!dm_table_contains(a.table, key)) unknown |= 1u << k;
        }
        for (uint32_t c = 0; c < sm.n_combos; ++c) {
            const uint32_t lo = sm.combo_off[c], hi = sm.combo_off[c + 1];
            uint64_t acc = dm_combo_seed(hi - lo);
            bool all = true;
            for (uint32_t j = lo; j < hi; ++j) {
                const uint32_t k = sm.combo_members[j];
                if (!((have >> k) & 1u)) { all = false; break; }
                acc = dm_combo_fold(acc, fpv[k]);
            }
            if (!all) continue;                                   // a missing member skips the combination
            const uint64_t key = dm_make_key(acc ? acc : 1ull, dm_field_salt(sm.n + c));
            if (train) dm_table_insert(a.table, key, &a.hdr->error);
            else if (!dm_table_contains(a.table, key)) unknown |= 1u << (sm.n + c);
        }
        if (!train) {
            const uint32_t cnt = (uint32_t)__popc(unknown);
            a.flags[r] = cnt ? 1 : 0;
            a.scores[r] = (float)cnt;
            a.masks[r] = unknown;
            if (cnt) {
                atomicAdd(&a.hdr->n_anomalies, 1ull);
                atomicAdd(a.stats + 3, 1ull);
                atomicAdd(a.stats + 4, (unsigned long long)cnt);
                uint32_t m = unknown;
                while (m) { const int k = __ffs(m) - 1; m &= m - 1; atomicAdd(a.stats + 8 + k, 1ull); }
            }
        } else {
            a.flags[r] = 0; a.scores[r] = 0.0f; a.masks[r] = 0;
        }
    }
}

// One CTA, after phase 2: bound[0] = the index just past the n_train-th well-formed record (n_records if the batch
// holds fewer), bound[1] = the well-formed records before it, i.e. the records trained.  Training counts well-formed
// records only, as the per-record path does (a malformed record raises before it takes a training slot).
__global__ void __launch_bounds__(256) dm_k_records_bound(const uint8_t* __restrict__ ok, uint32_t n_records,
                                                          uint32_t n_train, uint32_t* bound) {
    __shared__ uint32_t s_sum[256];
    const uint32_t tid = threadIdx.x;
    const uint32_t per = (n_records + 255) / 256;
    const uint32_t lo = tid * per < n_records ? tid * per : n_records;
    const uint32_t hi = lo + per < n_records ? lo + per : n_records;
    uint32_t s = 0;
    for (uint32_t r = lo; r < hi; ++r) s += ok[r];
    s_sum[tid] = s;
    __syncthreads();
    if (tid == 0) {
        uint32_t run = 0, t = 0;
        while (t < 256 && run + s_sum[t] < n_train) { run += s_sum[t]; ++t; }
        uint32_t b = n_records;
        if (t < 256) {
            uint32_t r = t * per;
            for (;; ++r)
                if (ok[r] && ++run == n_train) break;
            b = r + 1;
        }
        bound[0] = b;
        bound[1] = run;
    }
}
