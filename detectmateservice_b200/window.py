"""Multi-GPU plumbing: shard the record stream by line, one all-reduce per window.

One process per GPU (torch.distributed, NCCL between the GPUs of one node).  Detection is a
pure per-record lookup against read-only state, so the stream shards by record with no
data-path collective; the only exchange is, once per window, ONE sum-all-reduce of a small
uint64 buffer that carries

    words [0, 40)                       the statistics delta of the window (dm_stats_t layout)
    words 40 + r*(1+K) ..               rank r's segment: [count, key_0 .. key_{K-1}]

Rank r writes keys only into its own segment, so the sum is a concatenation: every rank
ends up with every rank's newly learnt keys (training windows) and the global statistics.
K = WINDOW_KEYS (65536) keys per rank per window; a rank that learnt more ships the rest in
further windows with keys (DeviceWindow.exchange drains them).  In steady-state detection the
buffer is just the 40 statistics words.

The device side of this (pack / merge kernels) is dm_window_export / dm_window_import of the
C ABI; this module holds the host side: record-aligned sharding of a message and a host
mirror of the buffer layout (used by the CPU tests of the N>1 path over gloo).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

STATS_WORDS = 40
WINDOW_KEYS = 1 << 16


def shard_bounds(buf, world: int) -> List[int]:
    """world+1 byte offsets cutting `buf` into `world` contiguous shards that start at record
    starts (each cut moved forward to just behind the next '\\n'); concatenating the shards'
    outputs in rank order preserves the global record order."""
    arr = np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf
    n = int(arr.size)
    cuts = [0]
    for r in range(1, world):
        p = max((n * r) // world, cuts[-1])
        if p >= n:
            cuts.append(n)
            continue
        if p > 0 and arr[p - 1] != 10:
            nl = np.flatnonzero(arr[p:] == 10)
            p = n if nl.size == 0 else p + int(nl[0]) + 1
        cuts.append(p)
    cuts.append(n)
    return cuts


def window_words(world: int, with_keys: bool, seg_keys: int = WINDOW_KEYS) -> int:
    """Words of a window buffer of `world` ranks with seg_keys keys per rank segment (the library's: WINDOW_KEYS)."""
    return STATS_WORDS + (world * (1 + seg_keys) if with_keys else 0)


def pack_window_host(stats_delta: Sequence[int], keys: Sequence[int], rank: int, world: int, with_keys: bool,
                     seg_keys: int = WINDOW_KEYS) -> np.ndarray:
    """Host mirror of dm_window_export's buffer (int64 view: the all-reduce is a two's
    complement sum, identical bit-for-bit to the uint64 sum)."""
    buf = np.zeros(window_words(world, with_keys, seg_keys), dtype=np.uint64)
    buf[:len(stats_delta)] = np.asarray(stats_delta, dtype=np.uint64)
    if with_keys:
        keys = np.asarray(keys, dtype=np.uint64)
        if keys.size > seg_keys:
            raise ValueError(f"{keys.size} keys learnt in one window, at most {seg_keys} can be exchanged")
        seg = STATS_WORDS + rank * (1 + seg_keys)
        buf[seg] = keys.size
        buf[seg + 1:seg + 1 + keys.size] = keys
    return buf.view(np.int64)


def unpack_window_host(buf: np.ndarray, world: int, with_keys: bool, seg_keys: int = WINDOW_KEYS
                       ) -> Tuple[np.ndarray, List[np.ndarray]]:
    """(global statistics delta, [keys of rank 0, keys of rank 1, ...]) of an all-reduced buffer."""
    u = np.asarray(buf).view(np.uint64)
    stats = u[:STATS_WORDS].copy()
    per_rank: List[np.ndarray] = []
    if with_keys:
        for r in range(world):
            seg = STATS_WORDS + r * (1 + seg_keys)
            cnt = int(u[seg])
            per_rank.append(u[seg + 1:seg + 1 + cnt].copy())
    return stats, per_rank


class DeviceWindow:
    """The per-window exchange of one rank's DeviceDetector (used by bench.py and by services
    launched one-per-GPU under torchrun)."""

    def __init__(self, det, rank: int, world: int, device):
        import torch
        self.det, self.rank, self.world = det, rank, world
        self.buf = torch.zeros(det.window_words(world, True), dtype=torch.int64, device=device)
        self.buf_stats = self.buf[:det.window_words(world, False)]

    def init_native(self, n_comms: int = 1) -> None:
        """Switch to the library's own NCCL communicator (one C call per window instead of
        export + torch.distributed.all_reduce + import; the id travels over torch.distributed)."""
        import torch
        import torch.distributed as dist
        dev = self.buf.device
        t = torch.zeros(128 * n_comms, dtype=torch.uint8, device=dev)
        if self.rank == 0:
            ids = b"".join(self.det.nccl_unique_id() for _ in range(n_comms))
            t.copy_(torch.frombuffer(bytearray(ids), dtype=torch.uint8))
        dist.broadcast(t, src=0)
        self.det.nccl_init(bytes(t.cpu().numpy().tobytes()), self.rank, self.world)
        self.native = True

    def exchange(self, with_keys: bool, stream_ptr: int) -> int:
        """One window on `stream_ptr`.  With keys, exchanges are repeated until no rank has learnt keys left that
        did not fit (more than WINDOW_KEYS since the previous window), so that every rank detects against every
        rank's keys; the ranks agree on the count through one MAX all-reduce per exchange.  Returns the number of
        exchanges."""
        n = 0
        while True:
            self._exchange_once(with_keys, stream_ptr)
            n += 1
            if not with_keys or not self._keys_pending():
                return n

    def _exchange_once(self, with_keys: bool, stream_ptr: int) -> None:
        if getattr(self, "native", False):
            self.det.window_allreduce(with_keys, stream_ptr)
            return
        import torch.distributed as dist
        buf = self.buf if with_keys else self.buf_stats
        self.det.window_export(buf.data_ptr(), self.rank, self.world, with_keys, stream_ptr)
        if self.world > 1:
            dist.all_reduce(buf, op=dist.ReduceOp.SUM)
        self.det.window_import(buf.data_ptr(), self.rank, self.world, with_keys, stream_ptr)

    def _keys_pending(self) -> bool:
        """Does any rank still hold keys its last export could not carry?  (At world 1: no collective.)"""
        pending = self.det.window_pending_keys()
        if self.world == 1:
            return pending > 0
        import torch
        import torch.distributed as dist
        t = torch.tensor([pending], dtype=torch.int64, device=self.buf.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return int(t.item()) > 0
