"""Shared helpers for the parity tests: fuzz inputs and oracle drivers."""
import numpy as np

from oracle.native import NativeOracle

FUZZ_KEYS = [b"a", b"ab", b"type", b"res", b"k1"]          # 5 distinct last bytes: candidate pre-filter off
FUZZ_KEYS_FEW = [b"a", b"ab", b"type", b"sa", b"ra"]        # 3 distinct last bytes: pre-filter on


def fuzz_lines(seed: int, n_lines: int, max_len: int = 600, alphabet: bytes = b"ab=  '\"typeresk1xq") -> bytes:
    """Random records over an alphabet rich in '=', space, both quote characters and the
    letters of the monitored keys -- stresses quote parity, field starts and duplicates."""
    r = np.random.Generator(np.random.PCG64(seed))
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    parts = []
    for _ in range(n_lines):
        mode = r.integers(0, 10)
        if mode == 0:
            ln = 0
        elif mode < 6:
            ln = int(r.integers(1, 64))
        elif mode < 9:
            ln = int(r.integers(64, 300))
        else:
            ln = int(r.integers(300, max_len + 1))
        parts.append(alpha[r.integers(0, alpha.size, ln)].tobytes())
    return b"\n".join(parts) + b"\n"


def lookalike_lines(seed: int, n_lines: int, keys=(b"key", b"type", b"res"), max_tokens: int = 260) -> bytes:
    """Records built from TOKENS rather than bytes: true fields, duplicates of them, quoted look-alikes
    (`q="x res=v y"`), apostrophe-led field starts, stray quotes that flip the parity for the rest of the
    record, dense runs of short fields (more than four '=' in 32 bytes) and long fillers -- up to a few KiB
    per record with dozens of candidates each.  Exercises the chained re-check of the stream kernel
    (dmx_verify_chain: carried state across batches, record starts inside a batch, fall-backs)."""
    r = np.random.Generator(np.random.PCG64(seed))
    vals = [b"aaa", b"bbb", b"cccc", b"success", b"quoted", b"xx1", b"xx2", b"new%d"]
    out = []
    for _ in range(n_lines):
        nt = int(r.integers(0, 8)) if r.random() < 0.6 else int(r.integers(8, max_tokens))
        toks = []
        dense_ok = r.random() < 0.04                               # (a dense row switches the chained re-check off around it)
        for _t in range(nt):
            u = r.random()
            if 0.64 <= u < 0.70 and not dense_ok:
                u = 0.9
            key = keys[int(r.integers(0, len(keys)))]
            v = vals[int(r.integers(0, len(vals)))]
            if b"%d" in v:
                v = v % int(r.integers(0, 40))
            if u < 0.30:
                toks.append(key + b"=" + v)
            elif u < 0.50:
                toks.append(b'q%d="v %s=%s x"' % (int(r.integers(0, 9)), key, v))
            elif u < 0.56:
                toks.append(b"'" + key + b"=" + v)
            elif u < 0.60:
                toks.append(b'"')                                  # stray quote: everything behind it is quoted
            elif u < 0.64:
                toks.append(b"x" + key + b"=" + v)                 # no field start
            elif u < 0.70:
                toks.append(b" ".join(b"%c=%d" % (97 + int(r.integers(0, 26)), int(r.integers(0, 10))) for _ in range(8)))
            elif u < 0.75:
                toks.append(key + b'="' + v + b' ' + v + b'"')     # quoted value with a space
            else:
                toks.append(b"f%d=%x" % (int(r.integers(0, 99)), int(r.integers(0, 1 << 24))))
        out.append(b" ".join(toks))
    return b"\n".join(out) + b"\n"


# ---------------------------------------------------------------------------------------------------------------------
# Byte-position sweep of the stream kernel's edges: 32-byte lanes, 1 KiB rows with the 16-byte slot prefix in front
# and the 64 bytes behind, the 32-byte value window, the message's first '=' and nbytes % 16.
# ---------------------------------------------------------------------------------------------------------------------
SWEEP_KEYS = [b"k", b"ab", b"res", b"type", b"acct_id", b"twelve_bytes", b"key_of_exactly_29_bytes_long"]
SWEEP_VALUE_LENS = (0, 1, 3, 4, 5, 31, 32, 33, 63, 64, 65, 200)
_SWEEP_ALPHA = b"abcdefghijklmnopqrstuvwxyz0123456789._-:/ABCDEFGH"


def _sweep_value(r, n: int, quoted: bool) -> bytes:
    v = bytearray(_SWEEP_ALPHA[i] for i in r.integers(0, len(_SWEEP_ALPHA), n))
    if quoted and n >= 8:
        # a quoted stretch holding spaces on both sides of the 32-byte window's end (byte 32 of the value)
        a = 0 if n < 40 else int(r.integers(0, 28))
        v[a] = v[n - 1] = 0x22
        for p in (29, 30, 31, 32, 33, 35):
            if a < p < n - 1 and r.random() < 0.6:
                v[p] = 0x20
    return bytes(v)


def _unknown_twin(v: bytes) -> bytes:
    """v with one byte changed near its end (behind the window for long values): unknown if only v was learnt."""
    if not v:
        return b"u"
    i = len(v) - 2 if v[-1] == 0x22 and len(v) >= 3 else len(v) - 1
    c = b"Z" if v[i] != ord("Z") else b"Y"
    return v[:i] + c + v[i + 1:]


def sweep_training(seed: int = 0, keys=SWEEP_KEYS):
    """(training message, {key: [learnt values]}): per key two values of every length in SWEEP_VALUE_LENS, one of
    them quoted where long enough; the empty value is learnt for every other key."""
    r = np.random.Generator(np.random.PCG64(seed))
    pool, recs = {}, []
    for i, k in enumerate(keys):
        vals = []
        for n in SWEEP_VALUE_LENS:
            if n == 0:
                if i % 2 == 0:
                    vals.append(b"")
                continue
            vals.append(_sweep_value(r, n, False))
            vals.append(_sweep_value(r, n, n >= 8))
        pool[k] = vals
        recs += [k + b"=" + v for v in vals]
    return b"\n".join(recs) + b"\n", pool


def _sweep_pick(r, pool, keys):
    k = keys[int(r.integers(0, len(keys)))]
    v = pool[k][int(r.integers(0, len(pool[k])))]
    return k, (v if r.random() < 0.5 else _unknown_twin(v))


def _sweep_gap(r, need: int) -> bytes:
    """need >= 1 bytes in front of a key: a value terminator, filler, and the key's field-start delimiter."""
    end = b"\n" if r.random() < 0.15 else b" "
    if need == 1:
        return end
    delim = b"'" if r.random() < 0.1 else b" "
    return end + b"x" * (need - 2) + delim


def sweep_messages(seed: int = 0, keys=SWEEP_KEYS, n_body: int = 6, body_bytes: int = 8000):
    """Detection messages for sweep_training(seed, keys): fields placed so that, over the list, the '=' falls on every
    residue mod 32 and on row offsets 0-17 and 1006-1023, the message's first '=' lies at bytes 1-4, every length of
    SWEEP_VALUE_LENS occurs (about half of them learnt values, the rest differ from a learnt one in one byte near the
    end), and messages end inside a value once for every nbytes % 16."""
    r = np.random.Generator(np.random.PCG64(seed + 1))
    _, pool = sweep_training(seed, keys)
    edges = list(range(18)) + list(range(1006, 1024))
    msgs = []
    # the message's first '=' at bytes 1..4 (the ring slot's prefix in front of the message reads as '\n')
    for k in keys:
        if len(k) <= 4:
            for lead in range(0, 5 - len(k)):
                kk, v = _sweep_pick(r, pool, [k])
                msgs.append(b" " * lead + kk + b"=" + v + b" k=" + _unknown_twin(v) + b"\n")
    # bodies: '=' at chosen residues mod 32 and at the row edges
    residue, edge = 0, 0
    for _m in range(n_body):
        b = bytearray()
        while len(b) < body_bytes:
            k, v = _sweep_pick(r, pool, keys)
            lo = len(b) + len(k) + (1 if b else 0)
            if r.random() < 0.5:
                q = lo + (edges[edge % len(edges)] - lo) % 1024
                edge += 1
            else:
                q = lo + int(r.integers(0, 24))
                q += (residue - q) % 32
                residue = (residue + 7) % 32
            if b:
                b += _sweep_gap(r, q - len(k) - len(b))
            else:
                b += b"x" * (q - len(k) - 1) + b" " if q > len(k) else b""
            b += k + b"=" + v
        msgs.append(bytes(b) + b"\n")
    # the message ends inside a value, for every nbytes % 16
    for m16 in range(16):
        k, v = _sweep_pick(r, pool, keys)
        head = b"k=1 " + b"y" * int(r.integers(0, 300)) + b"\n" + k + b"="
        tail = _sweep_value(r, 80, r.random() < 0.3)
        n = len(head) + 1 + (m16 - len(head) - 1) % 16 + 16 * int(r.integers(0, 4))
        msgs.append((head + tail)[:n])
    return msgs


# ---------------------------------------------------------------------------------------------------------------------
# Key-table limits: 32 monitored keys
# ---------------------------------------------------------------------------------------------------------------------
def _keys32():
    ks = {1: b"z", 2: b"cd", 3: b"q3q", 4: b"abcd", 5: b"xabcd", 6: b"yxabcd", 7: b"w_yxabcd"[1:],
          8: b"k\xc3\xa9y_0008", 13: b"long_key_abcd"}
    ks[8] = ks[8][:8]
    for n in range(1, 33):
        if n not in ks:
            tail = b"_end" if n in (20, 21, 27) else b"%04d" % n          # 20, 21, 27 share their last four bytes
            ks[n] = (b"f%02d_" % n + b"m" * 32)[:n - 4] + tail
    return [ks[n] for n in range(1, 33)]


KEYS32 = _keys32()
KEYS32_3BYTE = [bytes([97 + i // 6, 97 + (i * 5) % 26, 48 + i % 10]) for i in range(32)]     # 96 level-1 patterns


def keys32_lines(seed: int, n_lines: int, keys=KEYS32, known=None) -> bytes:
    """Records holding every one of the 32 keys (shuffled, values from `known` or fresh ones), plus look-alikes: a
    non-delimiter or an apostrophe in front of a key, keys at the record start, suffix keys inside longer keys."""
    r = np.random.Generator(np.random.PCG64(seed))
    out = []
    for i in range(n_lines):
        toks = []
        for j in r.permutation(len(keys)):
            k = keys[j]
            if known is not None and r.random() < 0.97:
                v = known[j][int(r.integers(0, len(known[j])))]
            else:
                v = b"v%d" % int(r.integers(0, 50))
            u = r.random()
            if u < 0.06:
                toks.append(b"x" + k + b"=" + v)                   # no field start
            elif u < 0.10:
                toks.append(b"'" + k + b"=" + v)                   # apostrophe starts a field
            elif u < 0.13:
                toks.append(b"'x" + k + b"=y" + v)
            toks.append(k + b"=" + v)
        out.append(b" ".join(toks))
    return b"\n".join(out) + b"\n"


def keys32_training(seed: int, keys=KEYS32, per_key: int = 6):
    """(training message, [[learnt values] per key])."""
    r = np.random.Generator(np.random.PCG64(seed))
    known = [[b"v%d" % int(x) for x in r.choice(50, per_key, replace=False)] for _ in keys]
    recs = [b" ".join(keys[j] + b"=" + known[j][i] for j in range(len(keys))) for i in range(per_key)]
    return b"\n".join(recs) + b"\n", known


# ---------------------------------------------------------------------------------------------------------------------
# Train/detect split inside one message
# ---------------------------------------------------------------------------------------------------------------------
def split_message(seed: int, n_records: int = 40, mean_len: int = 75, keys=(b"type", b"res", b"acct")) -> bytes:
    """About n_records * mean_len bytes of records with repeated values (what training teaches matters for the rest),
    the last one without its newline."""
    r = np.random.Generator(np.random.PCG64(seed))
    recs = []
    for i in range(n_records):
        toks = [b"%s=%s%d" % (k, k[:1], int(r.integers(0, 6))) for k in keys if r.random() < 0.8]
        pad = max(0, int(r.integers(mean_len // 2, 3 * mean_len // 2)) - sum(len(t) + 1 for t in toks))
        toks.insert(int(r.integers(0, len(toks) + 1)), b"p=" + b"y" * pad)
        recs.append(b" ".join(toks))
    return b"\n".join(recs)


def oracle_run(keys, train_msg: bytes, n_train: int, detect_msgs):
    """Train the C oracle on the first n_train records of train_msg (the rest of it is
    detected), then detect every message of detect_msgs.  Returns list of (flags, scores, masks)."""
    o = NativeOracle(keys)
    out = [o.process(train_msg, n_train, want_masks=True)]
    for m in detect_msgs:
        out.append(o.process(m, 0, want_masks=True))
    return o, out
