"""Wire-level ParserSchema generator for the record-mode tests.  TEST INFRASTRUCTURE.

Writes protobuf bytes field by field with its own varint and tag writer (it does not use
detectmateservice_b200/wire.py, whose encoder only ever writes canonical records).  Records come
in every encoding protobuf's runtime accepts -- shuffled and repeated fields, overlong varints,
map entries with missing, repeated or foreign fields, unknown and mistyped fields, multi-byte
UTF-8, long strings -- and a tagged mutation stage then breaks some of them.  Each record carries
the set of tags of what was done to it, so that a failure names the encoding; the oracle harness
(oracle/pbrecords.py) decides what is well-formed from protobuf's runtime itself, not from the tags.
"""
from __future__ import annotations

import random
from typing import List, Sequence, Set, Tuple

# ParserSchema field numbers
VERSION, PARSER_TYPE, PARSER_ID, EVENT_ID, TEMPLATE, VARIABLES = 1, 2, 3, 4, 5, 6
PARSED_LOG_ID, LOG_ID, LOG, LFV, RECEIVED_TS, PARSED_TS = 7, 8, 9, 10, 11, 12
STRING_FIELDS = (VERSION, PARSER_TYPE, PARSER_ID, TEMPLATE, PARSED_LOG_ID, LOG_ID, LOG)

# map keys the generator draws from: monitored keys of the test configs and their look-alikes
KEYS: List[bytes] = [b"k", b"use", b"user", b"users", b"K" * 64, b"K" * 63, "clé".encode(), b"", b"Time", b"level"]
# EventIDs: 0, small, negative (10-byte varint), and 2^31 + 5 (protobuf keeps its low 32 bits: -2147483643)
EVENT_IDS: List[int] = [0, 4, -7, (1 << 31) + 5, 1]
VALUES: List[bytes] = [b"a", b"b", b"", b"v", "é".encode(), "€x".encode(), "😀".encode(), b"a value"]
BAD_UTF8: List[Tuple[str, bytes]] = [("lone continuation", b"\x80"), ("overlong C0 80", b"\xc0\x80"),
                                     ("surrogate ED A0 80", b"\xed\xa0\x80"), ("above U+10FFFF F4 90 80 80", b"\xf4\x90\x80\x80"),
                                     ("FF", b"\xff"), ("cut 3-byte sequence", b"\xe2\x82")]


def varint(v: int, length: int = 0) -> bytes:
    """v as a varint (negative: 64-bit two's complement), padded to `length` bytes with overlong zero groups."""
    if v < 0:
        v += 1 << 64
    groups = []
    while True:
        groups.append(v & 0x7F)
        v >>= 7
        if not v:
            break
    groups += [0] * (length - len(groups))
    return bytes([g | 0x80 for g in groups[:-1]] + [groups[-1]])


def tag(field: int, wt: int, length: int = 0) -> bytes:
    return varint((field << 3) | wt, length)


def ld(field: int, payload: bytes, tag_len: int = 0, len_len: int = 0) -> bytes:
    return tag(field, 2, tag_len) + varint(len(payload), len_len) + payload


def frame(records: Sequence[bytes], r: random.Random = None, overlong_p: float = 0.0) -> bytes:
    """Length-delimited framing; with probability overlong_p a prefix is padded to 2..10 bytes."""
    out = bytearray()
    for rec in records:
        pad = r.randint(2, 10) if r is not None and r.random() < overlong_p else 0
        out += varint(len(rec), pad) + rec
    return bytes(out)


class Gen:
    """gen.record() -> (bytes, tags).  `novel` is the chance that a value is fresh (never seen before)."""

    def __init__(self, seed: int, novel: float = 0.05, mutate: float = 0.25, max_vars: int = 40, long_p: float = 0.01):
        self.r = random.Random(seed)
        self.novel, self.mutate_p, self.max_vars, self.long_p = novel, mutate, max_vars, long_p
        self.n = 0

    # ---------------------------------------------------------------- pieces
    def value(self) -> bytes:
        r = self.r
        if r.random() < self.long_p:                      # inner length varints of 1, 2 and 3 bytes
            n = r.choice([127, 128, 16383, 16384])
            unit = r.choice(["L", "é", "€", "😀"]).encode()
            body = unit * (n // len(unit))
            return body + b"L" * (n - len(body))
        if r.random() < self.novel:
            self.n += 1
            return ("new-%d-" % self.n).encode() + r.choice(VALUES)
        return r.choice(VALUES[:4]) if r.random() < 0.7 else r.choice(VALUES)

    def tlen(self) -> int:
        """tag length: canonical mostly, sometimes padded up to the 5 bytes protobuf accepts"""
        return self.r.randint(2, 5) if self.r.random() < 0.05 else 0

    def map_entry(self, tags: Set[str]) -> bytes:
        r = self.r
        key = r.choice(KEYS)
        k = ld(1, key, self.tlen())
        v = ld(2, self.value(), self.tlen())
        shape = r.random()
        if shape < 0.55:
            body = k + v
        elif shape < 0.62:
            body, _ = k, tags.add("entry: key only")
        elif shape < 0.67:
            body, _ = v, tags.add("entry: value only")
        elif shape < 0.74:
            body, _ = v + k, tags.add("entry: value before key")
        elif shape < 0.80:
            body, _ = ld(1, r.choice(KEYS)) + k + v + (ld(2, self.value()) if r.random() < 0.5 else b""), tags.add("entry: repeated key/value")
            if r.random() < 0.5:
                body = k + ld(2, self.value()) + v
        elif shape < 0.83:
            body, _ = b"", tags.add("entry: empty")
        else:
            foreign = r.choice([ld(3, b"q"), tag(3, 0) + varint(5), tag(1, 0) + varint(7), tag(2, 0) + varint(1),
                                tag(2, 5) + b"\0\0\0\0", tag(1, 1) + b"\0" * 8, ld((1 << 29) - 1, b"\xff\xfe"),
                                tag(9, 5) + b"abcd"])
            parts = [k, v, foreign]
            r.shuffle(parts)
            body, _ = b"".join(parts), tags.add("entry: foreign field")
        return ld(LFV, body, self.tlen())

    def unknown_field(self, tags: Set[str]) -> bytes:
        r = self.r
        f = r.choice([13, 15, 16, 100, 2047, 2048, (1 << 29) - 1, r.randint(13, (1 << 29) - 1)])
        wt = r.choice([0, 1, 2, 5])
        tags.add("unknown wt%d" % wt)
        if wt == 0:
            return tag(f, 0) + varint(r.choice([0, 1, 300, -1, 1 << 40]))
        if wt == 1:
            return tag(f, 1) + bytes(r.randrange(256) for _ in range(8))
        if wt == 5:
            return tag(f, 5) + bytes(r.randrange(256) for _ in range(4))
        return ld(f, bytes(r.randrange(256) for _ in range(r.randint(0, 12))))   # bytes, not checked for UTF-8

    def mistyped_field(self, tags: Set[str]) -> bytes:
        r = self.r
        tags.add("mistyped known field")
        return r.choice([tag(VARIABLES, 0) + varint(5), ld(EVENT_ID, b"\x01"), tag(LFV, 0) + varint(3),
                         tag(LFV, 5) + b"abcd", tag(VERSION, 0) + varint(1), tag(LOG, 1) + b"\0" * 8,
                         ld(RECEIVED_TS, b"\xff"), tag(VARIABLES, 5) + b"\xff\xff\xff\xff"])

    def event_id(self, tags: Set[str]) -> bytes:
        r = self.r
        e = r.choice(EVENT_IDS)
        if r.random() < 0.15 and e >= 0:
            tags.add("EventID overlong")
            return tag(EVENT_ID, 0) + varint(e, r.randint(len(varint(e)) + 1, 10))
        if r.random() < 0.05:
            tags.add("EventID 10th-byte overflow")               # bits past 64 are dropped
            return tag(EVENT_ID, 0) + bytes([0x80 | (e & 0x7F)]) + b"\x80" * 8 + bytes([r.choice([0x02, 0x7E, 0x7F])])
        return tag(EVENT_ID, 0) + varint(e)

    # ---------------------------------------------------------------- records
    def well_formed(self) -> Tuple[bytes, Set[str]]:
        r = self.r
        tags: Set[str] = set()
        items: List[bytes] = []
        if r.random() < 0.02:
            return b"", {"empty record"}
        if r.random() < 0.85:
            items.append(self.event_id(tags))
            if r.random() < 0.1:
                items.append(self.event_id(tags))
                tags.add("EventID repeated")
        nv = r.randint(0, self.max_vars) if r.random() < 0.15 else r.randint(0, 3)
        items += [ld(VARIABLES, self.value() if r.random() < 0.9 else b"", self.tlen()) for _ in range(nv)]
        items += [self.map_entry(tags) for _ in range(r.randint(0, 5))]
        for f in STRING_FIELDS:
            if r.random() < 0.3:
                items.append(ld(f, r.choice(VALUES) * r.randint(0, 4)))
        if r.random() < 0.3:
            items.append(tag(RECEIVED_TS, 0) + varint(r.choice([0, 1642723741, -5])))
        if r.random() < 0.25:
            items.append(self.unknown_field(tags))
        if r.random() < 0.15:
            items.append(self.mistyped_field(tags))
        if r.random() < 0.05:
            items.append(ld(LOG_ID, b"x") + ld(LOG_ID, b"y"))
            tags.add("singular string repeated")
        if r.random() < 0.4:
            r.shuffle(items)                                      # variables keep their relative order only by chance
            tags.add("shuffled")
        return b"".join(items), tags

    def mutate(self, rec: bytes, tags: Set[str]) -> bytes:
        r = self.r
        kind = r.choice(["cut", "flip", "utf8", "utf8", "field0", "bigtag", "varint11", "fixed_cut", "len_past",
                         "group", "tag6", "bad_wt"])
        if kind == "cut" and rec:
            i = r.randrange(len(rec))
            tags.add("cut at %d/%d" % (i, len(rec)))
            return rec[:i]
        if kind == "flip" and rec:
            i = r.randrange(len(rec))
            tags.add("flip byte %d" % i)
            return rec[:i] + bytes([rec[i] ^ r.randint(1, 255)]) + rec[i + 1:]
        if kind == "utf8":
            name, bad = r.choice(BAD_UTF8)
            val = b"ok" + bad + (b"" if name.startswith("cut") else b"tail")
            where = r.choice(["variables", "monitored map value", "map key", "log", "parserType", "dropped entry"])
            tags.add("invalid UTF-8 (%s) in %s" % (name, where))
            ins = {"variables": ld(VARIABLES, val), "monitored map value": ld(LFV, ld(1, r.choice(KEYS[:5])) + ld(2, val)),
                   "map key": ld(LFV, ld(1, val) + ld(2, b"v")), "log": ld(LOG, val), "parserType": ld(PARSER_TYPE, val),
                   "dropped entry": ld(LFV, ld(1, b"k") + ld(3, b"q") + ld(2, val))}[where]
            return self._insert(rec, ins)
        if kind == "field0":
            tags.add("field 0")
            return self._insert(rec, r.choice([b"\x00\x01", b"\x02\x01z", b"\x05abcd"]))
        if kind == "bigtag":
            hi = r.randint(32, 34)
            f = r.choice([VARIABLES, LFV])
            body = ld(1, b"k") + ld(2, b"z") if f == LFV else b"z"
            tags.add("tag (%d<<3|2) + 2^%d" % (f, hi))
            return self._insert(rec, varint(((f << 3) | 2) | (1 << hi)) + varint(len(body)) + body)
        if kind == "varint11":
            tags.add("11-byte varint")
            return self._insert(rec, tag(EVENT_ID, 0) + b"\xff" * 10 + b"\x01")
        if kind == "fixed_cut":
            w = r.choice([1, 5])
            tags.add("fixed%d cut short" % (64 if w == 1 else 32))
            return rec + tag(r.choice([13, EVENT_ID, VARIABLES]), w) + b"\0" * r.randint(0, 7 if w == 1 else 3)
        if kind == "len_past":
            n = r.randint(0, 5)
            tags.add("LEN past the record")
            return rec + tag(r.choice([VARIABLES, LFV, 13]), 2) + varint(n + r.randint(1, 300)) + b"a" * n
        if kind == "group":
            f = r.choice([EVENT_ID, VARIABLES, LFV, 13, 500])
            inner = r.choice([b"", tag(1, 0) + varint(1), ld(2, b"x")])
            tags.add("group")
            if r.random() < 0.3:                                  # inside a map entry
                return self._insert(rec, ld(LFV, ld(1, b"k") + tag(f, 3) + inner + tag(f, 4) + ld(2, b"v")))
            return self._insert(rec, tag(f, 3) + inner + tag(f, 4))
        if kind == "tag6":
            tags.add("6-byte tag")
            return self._insert(rec, tag(VARIABLES, 2, 6) + b"\x01z")
        tags.add("wire type 4/6/7")
        return self._insert(rec, tag(r.choice([13, VARIABLES]), r.choice([4, 6, 7])) + b"\x01z")

    def _insert(self, rec: bytes, field: bytes) -> bytes:
        """`field` at a field boundary of rec: the end, or the start, chosen at random (the record's own fields
        are not re-walked here)."""
        return rec + field if self.r.random() < 0.6 else field + rec

    def record(self) -> Tuple[bytes, Set[str]]:
        rec, tags = self.well_formed()
        if self.r.random() < self.mutate_p:
            rec = self.mutate(rec, tags)
        return rec, tags

    def records(self, n: int) -> Tuple[List[bytes], List[Set[str]]]:
        out = [self.record() for _ in range(n)]
        return [o[0] for o in out], [o[1] for o in out]
