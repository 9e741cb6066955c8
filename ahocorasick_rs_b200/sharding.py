"""Multi-GPU: one process per GPU, haystack batches sharded by contiguous index
ranges, the table replicated, no data-path collective during the scan.  The
only exchange is the gather of per-shard match lists (torch.distributed: NCCL
over NVLink on GPUs, gloo in the CPU tests); concatenation in rank order is
already the reference's order (SURVEY.md 8e).

The reference has nothing like this (one haystack per call, one core); the
semantics being preserved are simply "the batch result equals the per-haystack
results in haystack order"."""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import numpy as np


def partition_by_bytes(offsets: np.ndarray, world: int) -> List[Tuple[int, int]]:
    """Split haystacks [0, n) into `world` contiguous ranges with ~equal bytes.
    Returns [(lo, hi)] per rank (possibly empty ranges)."""
    n = len(offsets) - 1
    base = int(offsets[0])
    total = int(offsets[-1]) - base
    cuts = [0]
    for r in range(1, world):
        target = base + (total * r) // world
        # first haystack whose start is >= target
        idx = int(np.searchsorted(offsets[: n + 1], target, side="left"))
        cuts.append(min(max(idx, cuts[-1]), n))
    cuts.append(n)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


_GATHER_BUFS = {}   # (device, dtype) -> (send buffer, receive buffer) of gather_match_lists


def gather_match_lists(local, hay_base: int, group=None, dst: Optional[int] = None):
    """local: (k, 4) int32 or int64 tensor (haystack, pattern, start, end) with shard-local
    haystack ids.  Returns the global list (haystack ids rebased by each rank's
    hay_base) on every rank (dst=None) or on rank `dst` only (others get None).
    Two collectives: all_gather of the counts, then an all_gather padded to the longest list
    (no zero-filling, no per-rank copies: the bases are added in place on the gathered buffer)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = local.device
    meta = torch.tensor([local.shape[0], hay_base], dtype=torch.int64, device=dev)
    metas = torch.empty(world * 2, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(metas, meta, group=group)
    metas = metas.view(world, 2).tolist()
    counts = [int(c) for c, _ in metas]
    bases = [int(b) for _, b in metas]
    kmax = max(max(counts), 1)
    # Send and receive buffers are kept (grow-only) per device and dtype: a fresh multi-hundred-megabyte tensor per call
    # is handed to NCCL's stream and cannot be reused by the allocator until that stream has passed it, so every call
    # would cudaMalloc anew.
    key = (str(dev), local.dtype)
    bufs = _GATHER_BUFS.get(key)
    if bufs is None or bufs[0].numel() < kmax * 4 or bufs[1].numel() < world * kmax * 4:
        bufs = (torch.empty(kmax * 4 + kmax // 2, dtype=local.dtype, device=dev),
                torch.empty(world * (kmax * 4 + kmax // 2), dtype=local.dtype, device=dev))
        _GATHER_BUFS[key] = bufs
    padded = bufs[0][: kmax * 4].view(kmax, 4)
    padded[: local.shape[0]] = local
    everything = bufs[1][: world * kmax * 4]
    dist.all_gather_into_tensor(everything, padded.view(-1), group=group)
    everything = everything.view(world * kmax, 4)
    if dst is not None and rank != dst:
        return None
    parts = []
    for r in range(world):
        part = everything[r * kmax: r * kmax + counts[r]]
        if bases[r]:
            part[:, 0] += bases[r]
        parts.append(part)
    return parts[0].clone() if world == 1 else torch.cat(parts, dim=0)   # (a copy: the buffers are reused by the next call)


class MatchListGather:
    """The same exchange without touching the host: nothing here waits for the
    GPU, so a pipeline of scans keeps running.  Every rank contributes a fixed
    (cap + 1, 4) int32 block -- row 0 = (count, hay_base, complete flag, 0),
    then its first `cap` matches -- to ONE all_gather per call.  On a GPU the block
    is assembled by one kernel of the library (acb_pack_gather_block) and the
    exchange runs on a side stream: the caller's stream never waits for the
    collective of the step it just enqueued.  The caller cycles `slot` (and the
    scan's workspace: scan_device(..., ws_slot=slot)) through 0 .. slots-1; the scan that
    reuses a slot's workspace `slots` steps later is made to wait for that slot's
    exchange -- long finished by then (with eight ranks the collective's latency plus the
    skew between ranks exceeds one 0.2 ms step: four slots keep the scans running).  Call finish() before reading the result or
    timing the stream.  decode_gathered() turns a result into the ordered global
    list (that is where the host finally looks at the counts)."""

    def __init__(self, cap: int, device, group=None, slots: int = 2):
        import torch
        import torch.distributed as dist

        self.cap = cap
        self.group = group
        self.world = dist.get_world_size(group)
        self.device = device
        self.cuda = device.type == "cuda"
        self.slots = slots   # exchanges that may be in flight: the scan that reuses a slot waits for that slot's exchange
        self.blocks = [torch.zeros((cap + 1, 4), dtype=torch.int32, device=device) for _ in range(slots)]
        self.everything = [torch.empty(self.world * (cap + 1) * 4, dtype=torch.int32, device=device) for _ in range(slots)]
        self.side = torch.cuda.Stream(device=device) if self.cuda else None
        self.done = [None] * slots

    def __call__(self, matches, status, hay_base: int, slot: int = 0):
        """matches: the (capacity, 4) int32 output buffer of scan_device(sync=False); status: its
        8-entry int64 device status tensor ([0] = valid rows, [1] = complete flag).
        Returns the (world, cap + 1, 4) device tensor of this slot (reused two calls later)."""
        import torch
        import torch.distributed as dist

        block, everything = self.blocks[slot], self.everything[slot]
        if not self.cuda:
            # CPU tensors (gloo, tests): the same block, assembled with tensor ops
            k = min(self.cap, matches.shape[0])
            block[1: k + 1].copy_(matches[:k])
            lo = status.view(block.dtype)  # little-endian low words of the 64-bit counters
            block[0, 0] = lo[0]
            block[0, 2] = lo[2]
            block[0, 1] = hay_base
            dist.all_gather_into_tensor(everything, block.view(-1), group=self.group)
            return everything.view(self.world, self.cap + 1, 4)
        from . import _capi
        main = torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(main)  # the scan that produced `matches`
        with torch.cuda.stream(self.side):
            self.side.wait_event(ready)
            rc = _capi.lib().acb_pack_gather_block(status.data_ptr(), matches.data_ptr(), hay_base, self.cap, block.data_ptr(),
                                                   self.side.cuda_stream)
            if rc != _capi.ACB_OK:
                raise RuntimeError(_capi.last_error())
            dist.all_gather_into_tensor(everything, block.view(-1), group=self.group)
            ev = torch.cuda.Event()
            ev.record(self.side)
            self.done[slot] = ev
        # the NEXT scan writes the next slot's workspace, which the exchange `slots - 1` calls ago read
        nxt = self.done[(slot + 1) % self.slots]
        if nxt is not None:
            main.wait_event(nxt)
        return everything.view(self.world, self.cap + 1, 4)

    def finish(self):
        """Make the caller's stream wait for the exchanges in flight."""
        import torch

        if self.side is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.side)


def gather_match_lists_async(matches, status, hay_base: int, cap: int, group=None):
    """One-shot form of MatchListGather (allocates its buffers)."""
    return MatchListGather(cap, matches.device, group)(matches, status, hay_base)


def decode_gathered(gathered):
    """(world, cap + 1, 4) from gather_match_lists_async -> the global (k, 4) list in
    haystack order.  Raises if a rank's list did not fit its block."""
    import torch

    world, cap1, _ = gathered.shape
    heads = gathered[:, 0, :].tolist()
    parts = []
    for r in range(world):
        count, base, complete, _ = heads[r]
        if count > cap1 - 1 or not complete:
            raise RuntimeError(f"rank {r}: {count} matches do not fit the gather block of {cap1 - 1} (or its scan was incomplete)")
        part = gathered[r, 1: 1 + count].clone()
        part[:, 0] += int(base)
        parts.append(part)
    return torch.cat(parts, dim=0)


def scan_sharded(scan_fn: Callable, data: np.ndarray, offsets: np.ndarray, group=None, device=None):
    """Every rank holds the whole host batch (tests / small inputs): scan my
    shard with scan_fn(data_shard, offsets_shard) -> (k,4) int32 tensor on
    `device`, then gather.  Returns the full ordered match list on every rank."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    lo, hi = partition_by_bytes(offsets, world)[rank]
    sub_offs = offsets[lo: hi + 1] - offsets[lo]
    sub_data = data[offsets[lo]: offsets[hi]]
    local = scan_fn(sub_data, sub_offs.astype(np.int64))
    return gather_match_lists(local, lo, group=group)


def scan_sharded_single(scan_fn: Callable, data: np.ndarray, max_pattern_len: int, group=None, codepoints: bool = False, device=None):
    """ONE large haystack, overlapping search, across the ranks (SURVEY.md 8e).  Rank r owns
    the bytes [a_r, b_r) of a contiguous split and scans [a_r - halo, b_r) with
    halo = max_pattern_len - 1: the automaton state depends on no more than that, so the
    windows are independent; each rank keeps the matches that END in (a_r, b_r] (every match
    has exactly one such owner) and the lists are gathered in rank order, which is the
    reference's order (by end, then start, then pattern).

    scan_fn(window uint8 array) -> (k, 3) or (k, 4) integer tensor/array whose last three
    columns are (pattern, start, end) relative to the window -- byte offsets, or code point
    indexes when codepoints=True (the ranks then exchange how many continuation bytes each
    of them owns, to rebase the indexes).  Returns the global (k, 4) int64 tensor
    (0, pattern, start, end) on every rank.  Non-overlapping searches do not shard this way
    (restarts chain the ranges); the caller must not use this for them.  `device`: where the exchanged tensors
    live (None = CPU, for gloo; the CUDA device for NCCL)."""
    import torch
    import torch.distributed as dist

    dev = torch.device("cpu") if device is None else device
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n = len(data)
    a, b = (n * rank) // world, (n * (rank + 1)) // world
    halo = max(max_pattern_len - 1, 0)
    w0 = max(a - halo, 0)
    window = data[w0:b]
    got = scan_fn(window)
    got = got.cpu() if hasattr(got, "cpu") else torch.from_numpy(np.ascontiguousarray(got))
    got = got.to(torch.int64).reshape(got.shape[0], -1)
    local = torch.zeros((got.shape[0], 4), dtype=torch.int64)
    local[:, 1:] = got[:, -3:]
    shared = a - w0  # bytes of the window that belong to the previous ranks
    base = w0
    if codepoints:
        is_cont = (window & 0xC0) == 0x80
        # keep "byte end > shared" expressed in code points (see matcher._scan_one_large for the straddling case)
        shared_cp = shared - int(is_cont[:shared].sum())
        if shared < len(window) and is_cont[shared]:
            shared_cp -= 1
        keep = local[:, 3] > shared_cp if rank > 0 else torch.ones(local.shape[0], dtype=torch.bool)
        owned = torch.tensor([int(is_cont[shared:].sum())], dtype=torch.int64, device=dev)  # continuation bytes in [a, b)
        counts = torch.zeros(world, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(counts, owned, group=group)
        cont_before_a = int(counts[:rank].sum())
        cont_before_w0 = cont_before_a - int(is_cont[:shared].sum())
        base = w0 - cont_before_w0
    else:
        keep = local[:, 3] > shared if rank > 0 else torch.ones(local.shape[0], dtype=torch.bool)
    local = local[keep]
    local[:, 2] += base
    local[:, 3] += base
    # gather with 64-bit records (offsets of a multi-gigabyte haystack): counts first, then padded blocks
    cnt = torch.tensor([local.shape[0]], dtype=torch.int64, device=dev)
    cnts = torch.zeros(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(cnts, cnt, group=group)
    cnts = cnts.cpu()
    kmax = max(int(cnts.max()), 1)
    padded = torch.zeros((kmax, 4), dtype=torch.int64, device=dev)
    padded[: local.shape[0]] = local.to(dev)
    everything = torch.zeros(world * kmax * 4, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(everything, padded.view(-1), group=group)
    everything = everything.view(world, kmax, 4).cpu()
    return torch.cat([everything[r, : int(cnts[r])] for r in range(world)], dim=0)

