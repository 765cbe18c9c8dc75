"""Hand-written proto3 codec for the two messages on the detector's wire.

Schema (decoded from the descriptor the reference embeds in
/root/reference/container/fluentout/schemas_pb.rb:8; SURVEY.md Appendix A):

  ParserSchema    1 __version__ str   2 parserType str  3 parserID str   4 EventID int32
                  5 template str      6 variables rep str               7 parsedLogID str
                  8 logID str         9 log str        10 logFormatVariables map<str,str>
                  11 receivedTimestamp int32            12 parsedTimestamp int32
  DetectorSchema  1 __version__ str   2 detectorID str  3 detectorType str 4 alertID str
                  5 detectionTimestamp int32            6 logIDs rep str   8 score float
                  9 extractedTimestamps rep int32 (packed) 10 description str
                  11 receivedTimestamp int32            12 alertsObtain map<str,str>

The upstream parser stage produces ParserSchema, the downstream sink (fluentd,
container/fluentout/fluent.conf:4-17) parses one DetectorSchema per message.  No protobuf
runtime is needed on the hot path; tests cross-check this codec against protobuf's own.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Tuple


class WireError(ValueError):
    pass


def _read_varint(buf: bytes, pos: int) -> Tuple[int, int]:
    result = 0
    shift = 0
    n = len(buf)
    while True:
        if pos >= n:
            raise WireError("truncated varint")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 63:
            raise WireError("varint too long")


def _write_varint(out: bytearray, v: int) -> None:
    if v < 0:
        v += 1 << 64
    while v > 0x7F:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)


def _int32(v: int) -> int:
    v &= 0xFFFFFFFFFFFFFFFF
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v & 0x80000000 else v


def _write_str(out: bytearray, field: int, s) -> None:
    b = s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8")
    out.append((field << 3) | 2)
    _write_varint(out, len(b))
    out += b


def _write_map_entry(out: bytearray, field: int, k, v) -> None:
    e = bytearray()
    _write_str(e, 1, k)
    _write_str(e, 2, v)
    out.append((field << 3) | 2)
    _write_varint(out, len(e))
    out += e


# wire types expected per ParserSchema field number
_PARSER_LEN = {1, 2, 3, 5, 6, 7, 8, 9, 10}
_PARSER_VARINT = {4, 11, 12}
_PARSER_NAMES = {1: "__version__", 2: "parserType", 3: "parserID", 5: "template", 7: "parsedLogID", 8: "logID", 9: "log"}


def _read_tag(buf: bytes, pos: int) -> Tuple[int, int, int]:
    """(field, wire type, pos) as protobuf's runtime reads a tag: at most 5 bytes, below 2^32, field not 0."""
    start = pos
    tag, pos = _read_varint(buf, pos)
    if pos - start > 5 or tag >> 32:
        raise WireError("tag out of range")
    if tag >> 3 == 0:
        raise WireError("field number 0")
    return tag >> 3, tag & 7, pos


def _skip_field(buf: bytes, pos: int, end: int, wt: int) -> int:
    """Position after the payload of a field that is not read.  Groups (wire types 3/4) raise: proto3 cannot declare
    them, so a ParserSchema holding one is refused (protobuf's runtime would skip it)."""
    if wt == 0:
        _, pos = _read_varint(buf, pos)
    elif wt == 1:
        pos += 8
    elif wt == 5:
        pos += 4
    elif wt == 2:
        ln, pos = _read_varint(buf, pos)
        pos += ln
    else:
        raise WireError(f"unexpected wire type {wt}")
    if pos > end:
        raise WireError("field runs past the end")
    return pos


def _utf8(b: bytes) -> str:
    try:
        return b.decode("utf-8")
    except UnicodeDecodeError as e:
        raise WireError(f"string field is not valid UTF-8: {e}") from None


def decode_parser_schema(buf: bytes, strict: bool = True) -> Dict:
    """ParserSchema bytes -> dict with str values (EventID None when absent).
    Accepts and reads exactly what protobuf's runtime does (DESIGN.md section 5.3), except that a group raises:
    invalid UTF-8 in a string field, map key or value, field 0, a tag of 2^32 or more, or a payload running past the
    end raise WireError; a map entry holding anything but LEN fields 1 and 2 is dropped.
    strict: unknown fields / wrong wire types, at the top level or in a map entry, raise WireError too (used to tell a
    record from raw log lines); otherwise they are skipped like protobuf does."""
    rec: Dict = {"EventID": None, "variables": [], "logFormatVariables": {}, "logID": ""}
    pos, n = 0, len(buf)
    while pos < n:
        field, wt, pos = _read_tag(buf, pos)
        if wt == 2:
            ln, pos = _read_varint(buf, pos)
            end = pos + ln
            if end > n:
                raise WireError("length-delimited field runs past the end")
            if field == 10:
                k = v = ""
                foreign = False
                p = pos
                while p < end:
                    f2, w2, p = _read_tag(buf, p)
                    if w2 != 2 or f2 not in (1, 2):
                        if strict:
                            raise WireError("bad map entry")
                        p = _skip_field(buf, p, end, w2)
                        foreign = True
                        continue
                    l2, p = _read_varint(buf, p)
                    if p + l2 > end:
                        raise WireError("map entry runs past its end")
                    s = _utf8(buf[p:p + l2])
                    if f2 == 1:
                        k = s
                    else:
                        v = s
                    p += l2
                if not foreign:
                    rec["logFormatVariables"][k] = v
            elif field == 6:
                rec["variables"].append(_utf8(buf[pos:end]))
            elif field in _PARSER_NAMES:
                rec[_PARSER_NAMES[field]] = _utf8(buf[pos:end])
            elif strict:
                raise WireError(f"unexpected length-delimited field {field}")
            pos = end
        elif wt == 0:
            v, pos = _read_varint(buf, pos)
            if field == 4:
                rec["EventID"] = _int32(v)
            elif field == 11:
                rec["receivedTimestamp"] = _int32(v)
            elif field == 12:
                rec["parsedTimestamp"] = _int32(v)
            elif strict:
                raise WireError(f"unexpected varint field {field}")
        elif strict:
            raise WireError(f"unexpected wire type {wt} for field {field}")
        else:
            pos = _skip_field(buf, pos, n, wt)
    return rec


def looks_like_parser_schema(buf: bytes) -> bool:
    """A serialized ParserSchema starts with field 1..12 and walks cleanly; raw audit lines
    start with 't' (0x74 = field 14, wire type 4) and fail at the first byte."""
    if not buf or (buf[0] >> 3) not in range(1, 13):
        return False
    try:
        decode_parser_schema(buf, strict=True)
        return True
    except (WireError, IndexError):
        return False


def looks_like_delimited_parser_schemas(buf: bytes) -> bool:
    """varint length + a clean ParserSchema of exactly that length, at least for the first
    record (the batch framing of record mode)."""
    try:
        ln, pos = _read_varint(buf, 0)
    except (WireError, IndexError):
        return False
    if ln == 0 or pos + ln > len(buf):
        return False
    return looks_like_parser_schema(buf[pos:pos + ln])


def encode_parser_schema(rec: Dict) -> bytes:
    """dict -> ParserSchema bytes (used by tests and by the in-process demo pipeline)."""
    out = bytearray()
    _write_str(out, 1, rec.get("__version__", "1.0.0"))
    for field, name in ((2, "parserType"), (3, "parserID")):
        if name in rec:
            _write_str(out, field, rec[name])
    if rec.get("EventID") is not None:
        out.append(4 << 3)
        _write_varint(out, int(rec["EventID"]))
    if "template" in rec:
        _write_str(out, 5, rec["template"])
    for v in rec.get("variables") or []:
        _write_str(out, 6, v)
    for field, name in ((7, "parsedLogID"), (8, "logID"), (9, "log")):
        if name in rec:
            _write_str(out, field, rec[name])
    for k in sorted(rec.get("logFormatVariables") or {}):
        _write_map_entry(out, 10, k, rec["logFormatVariables"][k])
    for field, name in ((11, "receivedTimestamp"), (12, "parsedTimestamp")):
        if name in rec:
            out.append(field << 3)
            _write_varint(out, int(rec[name]))
    return bytes(out)


def encode_detector_schema(detector_id: str, detector_type: str, alert_id: str, detection_ts: int,
                           log_ids: List[str], score: float, extracted_ts: List[int], description: str,
                           received_ts: int, alerts: Dict[str, str], version: str = "1.0.0") -> bytes:
    out = bytearray()
    _write_str(out, 1, version)
    _write_str(out, 2, detector_id)
    _write_str(out, 3, detector_type)
    _write_str(out, 4, alert_id)
    out.append(5 << 3)
    _write_varint(out, int(detection_ts))
    for lid in log_ids:
        _write_str(out, 6, lid)
    out.append((8 << 3) | 5)
    out += struct.pack("<f", float(score))
    if extracted_ts:
        packed = bytearray()
        for t in extracted_ts:
            _write_varint(packed, int(t))
        out.append((9 << 3) | 2)
        _write_varint(out, len(packed))
        out += packed
    _write_str(out, 10, description)
    out.append(11 << 3)
    _write_varint(out, int(received_ts))
    for k in sorted(alerts):
        _write_map_entry(out, 12, k, alerts[k])
    return bytes(out)


def decode_detector_schema(buf: bytes) -> Dict:
    """DetectorSchema bytes -> dict (for tests and downstream consumers of the Python API)."""
    rec: Dict = {"logIDs": [], "extractedTimestamps": [], "alertsObtain": {}}
    names = {1: "__version__", 2: "detectorID", 3: "detectorType", 4: "alertID", 10: "description"}
    pos, n = 0, len(buf)
    while pos < n:
        tag, pos = _read_varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 2:
            ln, pos = _read_varint(buf, pos)
            end = pos + ln
            if end > n:
                raise WireError("field runs past the end")
            if field == 12:
                k = v = ""
                p = pos
                while p < end:
                    t, p = _read_varint(buf, p)
                    l2, p = _read_varint(buf, p)
                    s = buf[p:p + l2].decode("utf-8", "replace")
                    if t >> 3 == 1:
                        k = s
                    else:
                        v = s
                    p += l2
                rec["alertsObtain"][k] = v
            elif field == 6:
                rec["logIDs"].append(buf[pos:end].decode("utf-8", "replace"))
            elif field == 9:
                p = pos
                while p < end:
                    t, p = _read_varint(buf, p)
                    rec["extractedTimestamps"].append(_int32(t))
            elif field in names:
                rec[names[field]] = buf[pos:end].decode("utf-8", "replace")
            pos = end
        elif wt == 0:
            v, pos = _read_varint(buf, pos)
            if field == 5:
                rec["detectionTimestamp"] = _int32(v)
            elif field == 11:
                rec["receivedTimestamp"] = _int32(v)
            elif field == 9:
                rec["extractedTimestamps"].append(_int32(v))
        elif wt == 5:
            if field == 8:
                rec["score"] = struct.unpack("<f", buf[pos:pos + 4])[0]
            pos += 4
        elif wt == 1:
            pos += 8
        else:
            raise WireError(f"unexpected wire type {wt}")
    return rec


def frame_delimited(messages: List[bytes]) -> bytes:
    """varint-length-delimited stream (protobuf's writeDelimitedTo framing)."""
    out = bytearray()
    for m in messages:
        _write_varint(out, len(m))
        out += m
    return bytes(out)


def split_delimited(buf: bytes) -> List[bytes]:
    out, pos = [], 0
    while pos < len(buf):
        ln, pos = _read_varint(buf, pos)
        if pos + ln > len(buf):
            raise WireError("delimited frame runs past the end")
        out.append(buf[pos:pos + ln])
        pos += ln
    return out
