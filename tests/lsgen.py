"""Wire-level LogSchema generator and the rule R-log oracle for the LogSchema input tests.  TEST INFRASTRUCTURE.

Records are written field by field with pbgen's varint / tag writer, in the encodings protobuf's runtime accepts --
shuffled and repeated fields (a repeated `log` among them), overlong tags and lengths, unknown and mistyped fields --
and a mutation stage breaks some of them (groups, bad UTF-8 in each string field, cuts, field 0, 11-byte varints,
lengths past the end).  Texts come with trailing, inner and \\r\\n newlines.  What is well-formed is decided by
protobuf's runtime (oracle.schemas.LogSchema), not by the generator.

Oracle of R-log (DESIGN.md): decode every record with protobuf, drop the malformed and unusable ones, give every usable
text a '\\n', run the raw-line oracle on the joined message and scatter its results back to record order.
"""
from __future__ import annotations

import random
from typing import List, Optional, Sequence, Tuple

import numpy as np
from google.protobuf import message
from google.protobuf.unknown_fields import UnknownFieldSet

from oracle.schemas import LogSchema
from pbgen import BAD_UTF8, frame, ld, tag, varint

VERSION, LOG_ID, LOG, LOG_SOURCE, HOSTNAME = 1, 2, 3, 4, 5


def protobuf_text(rec: bytes) -> Tuple[Optional[bytes], Optional[str]]:
    """(text, logID) of one record as protobuf's runtime reads it and R-log shapes it; (None, None) when it is
    malformed (refused by protobuf, or holding a group) or unusable (a text of more than one line)."""
    m = LogSchema()
    try:
        m.ParseFromString(rec)
    except message.DecodeError:
        return None, None
    if any(f.wire_type == 3 for f in UnknownFieldSet(m)):
        return None, None
    text = m.log.encode("utf-8")
    if text.endswith(b"\n"):
        text = text[:-1]
    if b"\n" in text:
        return None, None
    return text, m.logID


def unwrap(records: Sequence[bytes]) -> Tuple[bytes, List[int], List[str]]:
    """(joined message of the usable texts, their record indices, every record's logID or None)."""
    parts, idx, ids = [], [], []
    for i, rec in enumerate(records):
        text, log_id = protobuf_text(rec)
        ids.append(log_id)
        if text is not None:
            parts.append(text + b"\n")
            idx.append(i)
    return b"".join(parts), idx, ids


def scatter(n: int, idx: Sequence[int], values, dtype) -> np.ndarray:
    out = np.zeros(n, dtype=dtype)
    if len(idx):
        out[np.asarray(idx, dtype=np.int64)] = np.asarray(values, dtype=dtype)[:len(idx)]
    return out


class Gen:
    """gen.record(text, log_id) -> (bytes, tags)."""

    def __init__(self, seed: int, mutate: float = 0.1, fuzz: float = 1.0):
        self.r = random.Random(seed)
        self.mutate_p = mutate
        self.fuzz = fuzz                                        # 0: canonical encodings only

    def _tlen(self) -> int:
        return self.r.randint(2, 5) if self.r.random() < 0.05 * self.fuzz else 0

    def _llen(self, n: int) -> int:
        return self.r.randint(len(varint(n)) + 1, 10) if self.r.random() < 0.05 * self.fuzz else 0

    def _str(self, field: int, value: bytes) -> bytes:
        return ld(field, value, self._tlen(), self._llen(len(value)))

    def well_formed(self, text: bytes, log_id: str) -> Tuple[bytes, set]:
        r, tags = self.r, set()
        items = [self._str(VERSION, b"1.0.0"), self._str(LOG_ID, log_id.encode()), self._str(LOG, text)]
        if r.random() < 0.5:
            items.append(self._str(LOG_SOURCE, b"/var/log/audit/audit.log"))
        if r.random() < 0.3:
            items.append(self._str(HOSTNAME, ("hôte-%d" % r.randint(0, 9)).encode()))
        f = self.fuzz
        if r.random() < 0.1 * f:
            items.append(r.choice([tag(13, 0) + varint(r.choice([0, 300, -1])), tag(99, 1) + b"\x01" * 8,
                                   tag(2047, 5) + b"\xff" * 4, ld(7, b"\xff\xfe not UTF-8, unknown field"),
                                   ld((1 << 29) - 1, b"")]))
            tags.add("unknown field")
        if r.random() < 0.05 * f:
            items.append(r.choice([tag(LOG, 0) + varint(5), tag(LOG_ID, 5) + b"abcd", tag(HOSTNAME, 1) + b"\0" * 8]))
            tags.add("mistyped known field")
        if r.random() < 0.4 * f:
            r.shuffle(items)
            tags.add("shuffled")
        if r.random() < 0.05 * f:
            # an earlier `log` that the last one overrides
            items.insert(0, self._str(LOG, b"decoy=1 type=DECOY"))
            tags.add("repeated log")
        return b"".join(items), tags

    def mutate(self, rec: bytes, tags: set) -> bytes:
        r = self.r
        kind = r.choice(["cut", "utf8", "field0", "varint11", "len_past", "group", "tag6", "inner_nl"])
        tags.add(kind)
        if kind == "cut" and rec:
            return rec[:r.randrange(len(rec))]
        if kind == "utf8":
            _name, bad = r.choice(BAD_UTF8)
            return rec + ld(r.choice([VERSION, LOG_ID, LOG, LOG_SOURCE, HOSTNAME]), b"ok" + bad)
        if kind == "field0":
            return b"\x02\x01z" + rec
        if kind == "varint11":
            return rec + tag(13, 0) + b"\xff" * 10 + b"\x01"
        if kind == "len_past":
            return rec + tag(LOG, 2) + varint(40) + b"abc"
        if kind == "group":
            return rec + tag(r.choice([LOG, 13]), 3) + tag(1, 0) + varint(1) + tag(r.choice([LOG, 13]), 4)
        if kind == "tag6":
            return rec + tag(LOG_ID, 2, 6) + b"\x01z"
        return rec + ld(LOG, b"first line\nsecond line")

    def record(self, text: bytes, log_id: str) -> Tuple[bytes, set]:
        rec, tags = self.well_formed(text, log_id)
        if self.r.random() < self.mutate_p:
            rec = self.mutate(rec, tags)
        return rec, tags

    def records(self, texts: Sequence[bytes], id_base: int = 0) -> List[bytes]:
        out = []
        for i, t in enumerate(texts):
            if self.r.random() < 0.03 * self.fuzz:
                t = t + b"\n"                                   # a reader that keeps line terminators
            elif self.r.random() < 0.01 * self.fuzz:
                t = t + b"\r\n"
            out.append(self.record(t, "id%d" % (id_base + i))[0])
        return out


def batch(records: Sequence[bytes], r: Optional[random.Random] = None) -> bytes:
    return frame(records, r, overlong_p=0.05 if r is not None else 0.0)
