"""R-tok -- sequential restatement of the raw audit-line tokenizer.  TEST INFRASTRUCTURE.

What it stands in for.  In the reference pipeline the detector never sees raw lines:
a MatcherParser stage (detectmatelibrary.parsers.template_matcher, configured at
/root/reference/tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88
with log_format ``type=<type> msg=audit(<Time>...): <Content>``) turns each line into a
ParserSchema whose ``logFormatVariables`` map the detector's ``header_variables``
read (docs/interfaces.md:138-204).  The CUDA path fuses that step: one message is N
'\\n'-terminated raw lines and every ``key=value`` field of a line is addressable as
a header variable.  The parser source is not in /root/reference, so this rule is
*defined here* (SURVEY.md section 8c, R-tok) and the CUDA tokenizer must reproduce
it byte for byte.

Rules (bytes, no decoding):
  L1  Records: every '\\n' ends a record (empty records count); a non-empty tail
      without '\\n' is a record too.  (src/service/core.py:190 counts the same way.)
  L2  in_quote(p) = parity of '"' (0x22) bytes in line[0:p).
  L3  A *separator* is a space (0x20) at p with in_quote(p) == 0.
  L4  p is a *field start* iff in_quote(p) == 0 and (p == 0 or line[p-1] is 0x20
      or line[p-1] is "'" (0x27)).  The single quote makes the inner k=v of
      ``msg='op=PAM:accounting acct="root" ...'`` addressable, matching the
      templates of tests/library_integration/audit_templates.txt:1-2,7-8.
  L5  A field start p yields a field iff the bytes from p up to the first '=' (at q)
      are non-empty and contain none of 0x20, 0x22, 0x27 (so the key is line[p:q]).
      Its value is line[q+1:e], e = first separator at or after q+1, else len(line).
  L6  Duplicate keys: the FIRST field with a given key wins.
  L7  ``Time`` (alert metadata only, never monitored): the first field with key
      ``msg`` whose value starts with ``audit(`` gives Time = value[6:j],
      j = first ':' or ')' after that, else end.
"""
from __future__ import annotations

from typing import Dict, Iterator, List, Tuple

SP, DQ, SQ, EQ, NL = 0x20, 0x22, 0x27, 0x3D, 0x0A


def split_records(buf: bytes) -> List[bytes]:
    """L1."""
    if not buf:
        return []
    parts = buf.split(b"\n")
    if parts[-1] == b"":
        parts.pop()
    return parts


def iter_fields(line: bytes) -> Iterator[Tuple[bytes, bytes, int]]:
    """Yield (key, value, q) for every field of the line in order (L2-L5)."""
    n = len(line)
    inq = 0
    p = 0
    while p < n:
        c = line[p]
        start = inq == 0 and (p == 0 or line[p - 1] == SP or line[p - 1] == SQ)
        if start:
            q = p
            ok = False
            while q < n:
                b = line[q]
                if b == EQ:
                    ok = q > p
                    break
                if b == SP or b == DQ or b == SQ:
                    break
                q += 1
            if ok:
                # value end: first separator at or after q+1 (quote parity continues
                # from the line start; the key holds no quote so in_quote(q+1)==0).
                e = q + 1
                vq = 0
                while e < n:
                    b = line[e]
                    if b == SP and vq == 0:
                        break
                    if b == DQ:
                        vq ^= 1
                    e += 1
                yield line[p:q], line[q + 1:e], q
        if c == DQ:
            inq ^= 1
        p += 1


def tokenize_line(line: bytes) -> Dict[bytes, bytes]:
    """First-occurrence field map of one line (L6)."""
    out: Dict[bytes, bytes] = {}
    for k, v, _ in iter_fields(line):
        if k not in out:
            out[k] = v
    return out


def line_time(line: bytes) -> bytes | None:
    """L7: the audit stamp's seconds part, or None.  Not a monitorable field: it only
    feeds DetectorSchema.extractedTimestamps of an alert."""
    for k, v, _ in iter_fields(line):
        if k == b"msg" and v.startswith(b"audit("):
            j = len(v)
            for idx in range(6, len(v)):
                if v[idx] in (0x3A, 0x29):
                    j = idx
                    break
            return v[6:j]
    return None
