"""The detector's state file (params.state_path): what a detector has learnt, kept across service restarts.

Layout, all integers little-endian:

    b"DMSTATE\\0"       magic, 8 bytes
    u32                 format version (FORMAT_VERSION)
    u32                 header length in bytes
    header              UTF-8 JSON object: component, key_signature, key_probe, n_seen, n_alerts, n_keys
    n_keys x u64        the known-set table's keys, strictly ascending, none zero

`key_signature` is everything a table key depends on (the component's key_signature()); `key_probe` is the key of one
fixed value (probe_key()), so a file written by a build with another fingerprint or salt does not match.  A file is
outside input: read_state() checks every length, the magic, the version and the key order, and raises ValueError
naming the first problem it finds.  write_state() replaces the file atomically: a failed write leaves the previous file
as it was.
"""
from __future__ import annotations

import json
import os
import struct
from typing import Any, Dict, Tuple

import numpy as np

MAGIC = b"DMSTATE\0"
FORMAT_VERSION = 1
HEADER_FIELDS = ("component", "key_signature", "key_probe", "n_seen", "n_alerts", "n_keys")
_PREFIX = struct.Struct("<8sII")


def probe_key() -> int:
    """dm_table_key(0, b"detectmate"): changes when the value fingerprint or the field salt does."""
    from . import _lib
    return int(_lib.load().dm_table_key(0, b"detectmate", 10))


def encode_state(header: Dict[str, Any], keys: np.ndarray) -> bytes:
    keys = np.ascontiguousarray(keys, dtype="<u8")
    hdr = dict(header, n_keys=int(keys.size))
    missing = [f for f in HEADER_FIELDS if f not in hdr]
    if missing:
        raise ValueError(f"state header lacks {', '.join(missing)}")
    if keys.size and (keys[0] == 0 or np.any(keys[1:] <= keys[:-1])):
        raise ValueError("state keys must be non-zero and strictly ascending")
    body = json.dumps(hdr, sort_keys=True, separators=(",", ":")).encode("utf-8")
    return _PREFIX.pack(MAGIC, FORMAT_VERSION, len(body)) + body + keys.tobytes()


def decode_state(blob: bytes) -> Tuple[Dict[str, Any], np.ndarray]:
    if len(blob) < _PREFIX.size:
        raise ValueError(f"state file truncated: {len(blob)} bytes, the fixed prefix alone takes {_PREFIX.size}")
    magic, version, hlen = _PREFIX.unpack_from(blob, 0)
    if magic != MAGIC:
        raise ValueError(f"not a detector state file: magic {magic!r}")
    if version != FORMAT_VERSION:
        raise ValueError(f"state file format version {version}, this build reads {FORMAT_VERSION}")
    if len(blob) < _PREFIX.size + hlen:
        raise ValueError(f"state file truncated: header of {hlen} bytes, {len(blob) - _PREFIX.size} present")
    try:
        hdr = json.loads(blob[_PREFIX.size:_PREFIX.size + hlen].decode("utf-8"))
    except (UnicodeDecodeError, ValueError) as e:
        raise ValueError(f"state file header is not UTF-8 JSON: {e}") from None
    if not isinstance(hdr, dict):
        raise ValueError("state file header is not a JSON object")
    missing = [f for f in HEADER_FIELDS if f not in hdr]
    if missing:
        raise ValueError(f"state file header lacks {', '.join(missing)}")
    for f in ("key_probe", "n_seen", "n_alerts", "n_keys"):
        if not isinstance(hdr[f], int) or isinstance(hdr[f], bool) or hdr[f] < 0:
            raise ValueError(f"state file header: {f} is not a non-negative integer")
    n = hdr["n_keys"]
    body = len(blob) - _PREFIX.size - hlen
    if body != 8 * n:
        raise ValueError(f"state file holds {body} key bytes, its header counts {n} keys ({8 * n} bytes)")
    keys = np.frombuffer(blob, dtype="<u8", count=n, offset=_PREFIX.size + hlen).astype(np.uint64)
    if n and keys[0] == 0:
        raise ValueError("state file holds a zero key")
    if n > 1 and np.any(keys[1:] <= keys[:-1]):
        raise ValueError("state file keys are not strictly ascending")
    return hdr, keys


def read_state(path: str) -> Tuple[Dict[str, Any], np.ndarray]:
    """(header, keys) of the file at path; ValueError if it is not a valid state file."""
    with open(path, "rb") as f:
        return decode_state(f.read())


def write_state(path: str, header: Dict[str, Any], keys: np.ndarray) -> None:
    """Write path.tmp beside path, flush and fsync it, rename it over path, then fsync the directory."""
    blob = encode_state(header, keys)
    tmp = path + ".tmp"
    try:
        with open(tmp, "wb") as f:
            f.write(blob)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        try:
            os.unlink(tmp)
        except OSError:
            pass
        raise
    fd = os.open(os.path.dirname(os.path.abspath(path)), os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)
