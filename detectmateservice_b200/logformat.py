"""Host-side mirror of the device's log_format / template matcher (csrc/dm_kernels_format.cuh).

Used by the component only to WORD the alerts of the (rare) anomalous records -- the value
text and the Time capture -- and to validate the configuration early; detection itself runs
on the device.  Same algorithm as the kernel (sequential earliest-occurrence search with an
end-anchored final literal), independent of the regular-expression oracle in oracle/rfmt.py.

Replaces, for those records, what detectmatelibrary.parsers.template_matcher.MatcherParser
puts into ParserSchema.logFormatVariables / EventID / variables
(/root/reference/tests/library_integration/test_pipe_filereader_matcher_nvd.py:74-88).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

_NAME_CHARS = frozenset(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_")
# the device's limits (csrc/dm_kernels_format.cuh); LogFormat applies them all
MAX_TEMPLATES = 63
MAX_CAPTURES = 32                    # per chain, whether it ends with a capture or with a literal
MAX_LITERAL_BYTES = 255              # per literal; template literals after R-norm
MAX_LITERALS = 512                   # over the log_format and all templates
POOL_BYTES = 4096                    # literal text over the log_format and all templates, each literal padded to 4-byte words

# R-norm (DESIGN.md): MatcherParser's params.remove_spaces / remove_punctuation / lowercase.  The same
# bits are passed to dm_set_format_ex; the device drops / folds the same bytes (DmFormat.norm_drop).
NORM_REMOVE_SPACES, NORM_REMOVE_PUNCTUATION, NORM_LOWERCASE = 1, 2, 4
_SPACES = bytes(range(0x09, 0x0E)) + b" "
_PUNCT = b"!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~"
_FOLD = bytes.maketrans(bytes(range(0x41, 0x5B)), bytes(range(0x61, 0x7B)))


def norm_flags(remove_spaces: bool = False, remove_punctuation: bool = False, lowercase: bool = False) -> int:
    return ((NORM_REMOVE_SPACES if remove_spaces else 0) | (NORM_REMOVE_PUNCTUATION if remove_punctuation else 0)
            | (NORM_LOWERCASE if lowercase else 0))


def normalise(text: bytes, flags: int) -> bytes:
    drop = (_SPACES if flags & NORM_REMOVE_SPACES else b"") + (_PUNCT if flags & NORM_REMOVE_PUNCTUATION else b"")
    return text.translate(_FOLD if flags & NORM_LOWERCASE else None, drop) if flags else text


class Chain:
    """L0 C0 L1 C1 ... L(n-1) [C(n-1)]"""
    __slots__ = ("literals", "ends_with_capture", "names")

    def __init__(self, literals: List[bytes], ends_with_capture: bool, names: List[str]):
        self.literals, self.ends_with_capture, self.names = literals, ends_with_capture, names

    @property
    def n_captures(self) -> int:
        return len(self.literals) if self.ends_with_capture else len(self.literals) - 1

    def match(self, text: bytes) -> Optional[List[bytes]]:
        lits, n, e = self.literals, len(self.literals), len(text)
        caps: List[bytes] = []
        pos = 0
        for i, lit in enumerate(lits):
            if i == 0:
                if not text.startswith(lit):
                    return None
                q = 0
            elif i == n - 1 and not self.ends_with_capture:
                q = e - len(lit)
                if q < pos or not text.endswith(lit):
                    return None
            else:
                q = text.find(lit, pos)
                if q < 0:
                    return None
            if i:
                caps.append(text[pos:q])
            pos = q + len(lit)
        if self.ends_with_capture:
            caps.append(text[pos:])
        elif pos != e:
            return None
        return caps


class _LiteralBudget:
    """The device's limits on literals over the log_format and all templates, checked literal by literal in the order
    dm_format_build adds them, with its reasons (csrc/dm_format_host.h)."""

    def __init__(self) -> None:
        self.n_lits = 0
        self.pool_words = 0

    def add(self, lit: bytes) -> None:
        if self.n_lits >= MAX_LITERALS:
            raise ValueError("too many literals over the log_format and the templates")
        if len(lit) > MAX_LITERAL_BYTES:
            raise ValueError("a literal between two captures is longer than 255 bytes")
        words = (len(lit) + 3) // 4
        if self.pool_words + words > POOL_BYTES // 4:
            raise ValueError("the literal text of log_format + templates exceeds 4096 bytes")
        self.pool_words += words
        self.n_lits += 1


def _parse(text: bytes, named: bool, flags: int = 0, budget: Optional[_LiteralBudget] = None) -> Chain:
    """One chain, checked as the device checks it.  Templates (named == False) are normalised literal by literal
    (R-norm: every literal is normalised, the wildcards stay)."""
    if budget is None:
        budget = _LiteralBudget()
    if b"\0" in text:
        raise ValueError("a NUL byte (the device's configuration strings end at the first one)")
    norm = (lambda s: s) if named else (lambda s: normalise(s, flags))
    lits: List[bytes] = []
    names: List[str] = []
    lit = bytearray()
    last_cap = False
    i = 0
    while i < len(text):
        end, name = -1, ""
        if text[i] == 0x3C:                                        # '<'
            if not named:
                if text[i:i + 3] == b"<*>":
                    end = i + 3
            else:
                j = i + 1
                while j < len(text) and text[j] in _NAME_CHARS:
                    j += 1
                if j > i + 1 and j < len(text) and text[j] == 0x3E:
                    end, name = j + 1, text[i + 1:j].decode()
        if end < 0:
            lit.append(text[i])
            i += 1
            last_cap = False
            continue
        if last_cap:
            raise ValueError("two captures with nothing between them")
        front = norm(bytes(lit))
        if lits and front == b"":
            raise ValueError("normalisation leaves nothing between two wildcards")
        budget.add(front)                                          # the literal in front of this capture (L0 may be empty)
        lits.append(front)
        lit = bytearray()
        names.append(name)
        last_cap = True
        i = end
    final = norm(bytes(lit))
    ends = last_cap or (not named and flags != 0 and bool(lits) and final == b"")   # `... <*>'` normalised: runs to the end
    if not ends:
        budget.add(final)                                          # the final literal (or the whole text)
        lits.append(final)
    if (len(lits) if ends else len(lits) - 1) > MAX_CAPTURES:
        raise ValueError("more than %d captures in one log_format / template" % MAX_CAPTURES)
    return Chain(lits, ends, names)


def _b(x) -> bytes:
    return x if isinstance(x, bytes) else str(x).encode("utf-8")


class LogFormat:
    """Raises ValueError on every configuration the device rejects, in dm_format_build's order and with its reasons,
    so that a bad configuration fails where the component is constructed rather than at its first message."""

    def __init__(self, log_format, templates: Sequence = (), content_name: str = "Content", flags: int = 0) -> None:
        self.source = _b(log_format).decode("utf-8")
        self.template_sources = [_b(t) for t in templates]
        self.flags = int(flags)
        self.content_name = content_name
        if b"\0" in _b(content_name):
            raise ValueError("content_name: a NUL byte (the device's configuration strings end at the first one)")
        budget = _LiteralBudget()
        try:
            self.header = _parse(_b(log_format), named=True, budget=budget)
        except ValueError as e:
            raise ValueError("log_format: %s" % e) from None
        for i, n in enumerate(self.header.names):
            if n in self.header.names[:i]:
                raise ValueError("log_format: capture <%s> appears twice" % n)
        if self.template_sources and content_name not in self.header.names:
            raise ValueError(f"templates given but log_format has no <{content_name}> capture")
        self.templates = []
        for t, src in enumerate(self.template_sources):
            try:
                if t >= MAX_TEMPLATES:
                    raise ValueError("too many templates (at most %d)" % MAX_TEMPLATES)
                self.templates.append(_parse(src, named=False, flags=self.flags, budget=budget))
            except ValueError as e:
                raise ValueError("template %d: %s" % (t, e)) from None

    def parse(self, line: bytes) -> Optional[Tuple[int, List[bytes], Dict[str, bytes]]]:
        """(EventID, variables, header variables) of one record, None if log_format does not match."""
        caps = self.header.match(line)
        if caps is None:
            return None
        lfv = dict(zip(self.header.names, caps))
        content = lfv.get(self.content_name)
        if content is not None:
            content = normalise(content, self.flags)             # variables are slices of the normalised text
            for t, ch in enumerate(self.templates):
                v = ch.match(content)
                if v is not None:
                    return t, v, lfv
        return -1, [], lfv


def load_templates(path: str) -> List[bytes]:
    """One template per non-empty line (params.path_templates of the reference parser config)."""
    with open(path, "rb") as f:
        return [ln for ln in f.read().split(b"\n") if ln.strip()]
