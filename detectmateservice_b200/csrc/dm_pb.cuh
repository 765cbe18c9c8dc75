// dm_pb.cuh -- the protobuf wire-format primitives the device walks records with: varints, tags as protobuf's
// runtime reads them, skipping a field by wire type, strict UTF-8.  Shared by the ParserSchema walk
// (dm_kernels_records.cuh) and the LogSchema walk (dm_kernels_logs.cuh), so that both refuse exactly the same
// records (DESIGN.md section 5.3).
#pragma once
#include "dm_device.cuh"

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
