"""Host-side mirror of the reference's Python API on top of the C ABI.

Reference being mirrored: /root/reference/src/lib.rs (PyO3 classes
``AhoCorasick`` 29-33/134-273, ``BytesAhoCorasick`` 360-435, enums 91-128) and
pysrc/ahocorasick_rs/ahocorasick_rs.pyi.  Same names, argument meaning and
error behaviour; the scan itself runs in the sm_90a kernels behind
include/acb200.h.  There is no CPU fallback: without the CUDA library or a
CUDA device every search raises.

Additions next to the drop-in methods (the reference API is one haystack per
call): ``find_matches_as_indexes_batch`` and ``scan_device`` for batches that
are already device resident; ``is_match`` / ``is_match_batch`` /
``is_match_device``, the crate's ``AhoCorasick::is_match`` per haystack;
``find_first`` / ``find_first_batch`` / ``find_first_device``, the crate's
``AhoCorasick::find`` per haystack; ``count_matches`` / ``count_matches_batch`` /
``count_matches_device``, the length of each haystack's match list without the list;
``count_matches_by_pattern`` / ``count_matches_by_pattern_batch`` /
``count_matches_by_pattern_device``, how many matches each pattern has over a batch.

``TokenAhoCorasick`` is the same API over token-id sequences (uint16 / int32 / int64): the ids are encoded into a
self-synchronising 3-byte format (include/acb200.h) and searched as bytes, positions divided by 3.  Its
``completing_tokens`` / ``completing_tokens_batch`` / ``completing_tokens_device`` and ``mask_completing_tokens_`` give
the next ids that would complete a pattern (a bad-words logits processor) from a token-level kernel of their own, and
``bias_completing_tokens_`` adds a bias per pattern to them (a sequence-bias logits processor).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import enum
import threading
from typing import Iterable, Optional, Sequence

import numpy as np

from . import _capi


class MatchKind(enum.Enum):
    """reference: src/lib.rs:92-98"""
    Standard = 0
    LeftmostFirst = 1
    LeftmostLongest = 2


class Implementation(enum.Enum):
    """reference: src/lib.rs:111-118.  Here, as there, a table-format choice that never changes results
    (tests/test_ac.py:22-56): DFA = the dense transition table (walked by the staged / L2 kernels when the data
    suits them), the two NFA values = the compact sieve image (filters + reverse trie, csrc/sieve.h); None = the
    library decides from a profile of the data."""
    NoncontiguousNFA = 0
    ContiguousNFA = 1
    DFA = 2


_TRACE = bool(__import__("os").environ.get("ACB200_TRACE"))


def _torch():
    import torch
    return torch


def _require_cuda():
    torch = _torch()
    if not torch.cuda.is_available():
        raise RuntimeError("ahocorasick_rs_b200 needs a CUDA device: the scan has no CPU fallback")
    return torch


def _count_cont(x) -> int:
    """UTF-8 continuation bytes (10xxxxxx) in a uint8 numpy array or torch tensor."""
    return int(((x & 0xC0) == 0x80).sum())


def scan_in_windows(scan_window, hay, window_bytes: int, halo: int, codepoints: bool):
    """An OVERLAPPING search over one haystack too large for one call, as independent windows that share `halo` =
    max_pattern_len - 1 bytes (what ends at a position depends on no more than that).  scan_window(window) returns the
    window's matches as int64 rows (haystack, pattern, start, end), window-relative, byte offsets or code point indexes,
    sorted by end.  Every window keeps the matches that END beyond the bytes it shares with its predecessor (those were
    reported, whole, by the predecessor) -- a suffix of its sorted rows --, rebased to the haystack.  `hay` is a uint8
    numpy array or torch tensor; returns the list of per-window row blocks, in order (concatenated they are in the
    reference's order)."""
    parts = []
    cont_before = 0  # continuation bytes before the window start (code point indexes)
    counted = 0      # ... counted up to here
    for w0, w1 in _windows(len(hay), window_bytes, halo):
        if codepoints:
            for a in range(counted, w0, 1 << 28):  # count in slices: the mask is a temporary of the slice's size
                cont_before += _count_cont(hay[a:min(a + (1 << 28), w0)])
            counted = w0
        window = hay[w0:w1]
        part = scan_window(window)
        if w0 > 0 and part.shape[0]:
            cut = halo
            if codepoints:
                # the same cut in code points: ends are character boundaries, so "byte end > halo" is "code point
                # end > code points that start before byte `halo`" -- minus one when a character straddles that
                # byte (its end is beyond the shared bytes although no new character starts in between)
                cut = halo - _count_cont(window[:halo])
                if halo < len(window) and (int(window[halo]) & 0xC0) == 0x80:
                    cut -= 1
            ends = part[:, 3]
            if hasattr(ends, "contiguous"):   # torch: the rows are sorted by end, the kept ones are a suffix
                import torch
                k0 = int(torch.searchsorted(ends.contiguous(), torch.tensor([cut], dtype=ends.dtype, device=ends.device), right=True).item())
            else:
                k0 = int(np.searchsorted(ends, cut, side="right"))
            part = part[k0:]
        base = (w0 - cont_before) if codepoints else w0
        if base:
            part[:, 2] += base
            part[:, 3] += base
        parts.append(part)
    return parts


def _windows(total_len: int, limit: int, halo: int):
    """The windows [w0, w1) of `limit` bytes at most that cover a haystack of total_len bytes, in order, each sharing
    `halo` bytes (max_pattern_len - 1) with its predecessor: every match lies inside one of them whole.  None for an
    empty haystack.  ValueError when limit <= halo (the windows would not advance)."""
    step = limit - halo
    if step <= 0:
        raise ValueError("window smaller than the longest pattern")
    w0 = 0
    while w0 < total_len:
        w1 = min(w0 + limit, total_len)
        yield w0, w1
        if w1 == total_len:
            return
        w0 += step


def _haystack_runs(offsets, limit: int):
    """Cuts a batch (offsets: int64 tensor (n + 1,)) that one call cannot take into calls, in haystack order: yields
    (h, h1, start, end, large), haystacks [h, h1) at bytes [start, end).  large = False: the longest run of whole
    haystacks from h that fits `limit` bytes and stops before an oversized one (at least one haystack; zero-byte runs
    too).  large = True: the single haystack h (h1 = h + 1) of more than `limit` bytes.  The host reads a few scalars
    of `offsets` per item and nothing else."""
    torch = _torch()
    n = offsets.numel() - 1
    if n <= 0:
        return
    lens = offsets[1:] - offsets[:-1]
    oversized = bool((lens > limit).any().item())
    h = 0
    while h < n:
        start = int(offsets[h].item())
        if oversized:
            size = int(lens[h].item())
            if size > limit:
                yield h, h + 1, start, start + size, True
                h += 1
                continue
        h1 = int(torch.searchsorted(offsets, torch.tensor([start + limit], dtype=torch.int64, device=offsets.device), right=True).item()) - 1
        h1 = max(h + 1, min(h1, n))
        if oversized:
            big = torch.nonzero(lens[h:h1] > limit)
            if big.numel():
                h1 = h + int(big[0].item())
        yield h, h1, start, int(offsets[h1].item()), False
        h = h1


def _pack_host(buf, chunks):
    """Lays bytes-like chunks (one per haystack) out for one host->device copy: the n + 1 int64 offsets, then the bytes
    from the first 512-byte boundary after them.  buf(nbytes) returns the uint8 numpy buffer to write, of at least
    nbytes.  -> (offsets, a numpy array of its own; head; total_bytes): the bytes are at buf[head:head + total_bytes]."""
    n = len(chunks)
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.fromiter((len(c) for c in chunks), dtype=np.int64, count=n), out=offs[1:])
    total_bytes = int(offs[-1])
    head = (8 * (n + 1) + 511) & ~511   # the offsets, then the bytes at a 512-byte boundary of the buffer
    hv = buf(head + total_bytes)
    hv[:8 * (n + 1)].view(np.int64)[:] = offs
    if n == 1:
        hv[head:head + total_bytes] = np.frombuffer(chunks[0], dtype=np.uint8)
    elif total_bytes:
        hv[head:head + total_bytes] = np.frombuffer(b"".join(chunks), dtype=np.uint8)
    return offs, head, total_bytes


def _check(rc):
    if rc != _capi.ACB_OK:
        raise RuntimeError(_capi.last_error())


# last_stats["paths"] of a table-walker scan: the branches its epilogue took (kPath* in csrc/capi.cu).  They never
# change results; tests check them to know that an input reached the path it was made for.
PATH_FAR_CP = 1      # code points: prefix sum of every segment's continuation bytes (a haystack spans > 8 segments)
PATH_SEARCH = 2      # per-haystack offsets by binary search (more than 4 records per haystack, or an incomplete list)
PATH_REPAIRED = 4    # some speculated segment start was wrong and the repair pass ran


class PatternSets:
    """Pattern sets of one automaton on one device: G subsets of its pattern ids, packed once into a bitset of G rows of
    ceil(P / 32) u32 words (bit p % 32 of word p // 32 of row g = pattern p is in set g).  Made by ``pattern_sets`` of
    the classes; a query given ``pattern_sets=ps, set_index=idx`` searches haystack i for the patterns of set idx[i]
    only, and returns exactly what an automaton built from those patterns (same match kind, same relative order)
    would return, with the full automaton's pattern ids."""

    def __init__(self, ac: "_Automaton", sets, device=None):
        torch = _torch()
        P = ac.n_patterns
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if torch.is_tensor(sets):
            if sets.dtype != torch.bool or sets.dim() != 2 or sets.shape[1] != P:
                raise ValueError(f"a tensor of pattern sets must be a bool tensor of shape (G, {P})")
            mask = sets.to(device)
        else:
            rows = [list(s) for s in sets]
            mask = np.zeros((len(rows), P), dtype=bool)
            for g, ids in enumerate(rows):
                for p in ids:
                    if isinstance(p, bool) or not isinstance(p, (int, np.integer)):
                        raise ValueError(f"set {g}: pattern ids must be ints, not {type(p).__name__}")
                    if not 0 <= int(p) < P:
                        raise ValueError(f"set {g}: pattern id {int(p)} is outside [0, {P})")
                    mask[g, int(p)] = True
            mask = torch.from_numpy(mask).to(device)
        if mask.shape[0] < 1:
            raise ValueError("pattern sets: at least one set is needed")
        self._ac = ac
        self.device = device
        self.n_sets = int(mask.shape[0])
        self.words = max((P + 31) // 32, 1)
        self.bits = self.pack(mask, self.words)

    @staticmethod
    def pack(mask, words: int):
        """(G, P) bool tensor -> (G, words) int32 tensor, the u32 bitset rows (torch ops on the mask's device)."""
        torch = _torch()
        G, P = mask.shape
        padded = torch.zeros((G, words * 32), dtype=torch.int64, device=mask.device)
        padded[:, :P] = mask.to(torch.int64)
        weights = torch.bitwise_left_shift(torch.ones(32, dtype=torch.int64, device=mask.device), torch.arange(32, device=mask.device))
        w = (padded.view(G, words, 32) * weights).sum(dim=2)
        return torch.where(w >= (1 << 31), w - (1 << 32), w).to(torch.int32).contiguous()


def _filter_args(ac: "_Automaton", pattern_sets, set_index, n: int, dev):
    """Checks a device call's (pattern_sets, set_index) -> the filter the internal paths carry: None, or
    (PatternSets, contiguous int32 / int64 index tensor (n,))."""
    flt = _filter_shape_args(ac, pattern_sets, set_index, n, dev)
    if flt is not None and n:
        lo, hi = (int(v) for v in _torch().stack(_torch().aminmax(set_index)).tolist())
        if lo < 0 or hi >= pattern_sets.n_sets:
            raise ValueError(f"set_index values must lie in [0, {pattern_sets.n_sets}); found [{lo}, {hi}]")
    return flt


def _filter_shape_args(ac: "_Automaton", pattern_sets, set_index, n: int, dev):
    """_filter_args without reading set_index back: everything it checks but the index values, so the call neither
    synchronises nor allocates (for a contiguous index).  The kernels give an index outside [0, n_sets) its defined
    meaning: the row admits no pattern."""
    torch = _torch()
    if pattern_sets is None and set_index is None:
        return None
    if pattern_sets is None or set_index is None:
        raise ValueError("pattern_sets and set_index go together: give both or neither")
    if not isinstance(pattern_sets, PatternSets) or pattern_sets._ac is not ac:
        raise ValueError("pattern_sets must come from this automaton's pattern_sets()")
    if pattern_sets.device != dev:
        raise ValueError(f"pattern_sets live on {pattern_sets.device}, the data on {dev}")
    if (not torch.is_tensor(set_index) or set_index.dtype not in (torch.int32, torch.int64) or set_index.dim() != 1 or
            set_index.shape[0] != n or set_index.device != dev):
        raise ValueError(f"set_index must be an int32 or int64 tensor of shape ({n},) on {dev}")
    return pattern_sets, set_index.contiguous()


def _filter_struct(flt):
    """The acb_pattern_filter of an internal filter (None: no filter, a NULL pointer)."""
    if flt is None:
        return None
    ps, idx = flt
    f = _capi.PatternFilter()
    f.dev_set_bits = ps.bits.data_ptr()
    f.n_sets = ps.n_sets
    f.dev_set_index = idx.data_ptr() if idx.numel() else ps.bits.data_ptr()
    f.index_bytes = idx.element_size()
    return C.byref(f)


def _filter_slice(flt, a: int, b: int):
    return None if flt is None else (flt[0], flt[1][a:b])


def _host_sets(ac: "_Automaton", patterns, n: int, dev):
    """A host call's patterns= -> an internal filter for its n haystacks: one set per haystack (n > 1: `patterns` holds
    one iterable per haystack; n == 1 and single: the iterable itself)."""
    torch = _torch()
    ps = PatternSets(ac, patterns, dev)
    if ps.n_sets != n:
        raise ValueError(f"patterns= needs one set of pattern ids per haystack: {n} haystacks, {ps.n_sets} sets")
    return ps, torch.arange(n, dtype=torch.int32, device=dev)


class _Automaton:
    """Owns the host automaton handle, its device image and a growable device
    workspace.  Shared by both public classes."""

    def __init__(self, pattern_bytes: Sequence[bytes], matchkind: MatchKind, implementation: Optional[Implementation]):
        L = _capi.lib()
        n = len(pattern_bytes)
        offs = np.zeros(n + 1, dtype=np.uint64)
        if n:
            np.cumsum(np.fromiter((len(p) for p in pattern_bytes), dtype=np.uint64, count=n), out=offs[1:])
        blob = np.frombuffer(b"".join(pattern_bytes) or b"\0", dtype=np.uint8)
        h = C.c_void_p()
        impl = -1 if implementation is None else implementation.value
        rc = L.acb_build(blob.ctypes.data, offs.ctypes.data, n, matchkind.value, impl, C.byref(h))
        if rc != _capi.ACB_OK:
            raise ValueError(_capi.last_error())
        self._h = h
        self._L = L
        self.matchkind = matchkind
        self.implementation = implementation
        self.n_patterns = n
        self.num_states = int(L.acb_num_states(h))
        self.num_columns = int(L.acb_num_columns(h))
        self.max_pattern_len = int(L.acb_max_pattern_len(h))
        self._images = {}      # device index -> uint8 tensor
        self._sieves = {}      # device index -> (uint8 tensor, SieveDesc)
        self._completions = {}   # device index -> (uint8 tensor, CompletionsDesc): token-format patterns only
        self._hot = {}         # device index -> dict(tensor, rows, reprofile, calls, backoff)
        self._ws = {}          # (device index, slot) -> dict of tensors
        self._small = {}       # device index -> the small-call context
        self._hit_row_words = 0   # hits_device: the counter-row words the largest call so far needed
        self.last_stats = {}
        self._lock = threading.RLock()   # (re-entered: any_device's table-walker path scans with scan_device under it)
        self._host_lock = threading.RLock()   # host-buffer calls: staging buffer + workspaces until the results are on the host

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self._L.acb_free(h)
            self._h = None

    # ---- device residency ---------------------------------------------------
    def image(self, device):
        """The flat tables on `device` (uploaded once, then cached)."""
        torch = _require_cuda()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        img = self._images.get(idx)
        if img is None:
            nbytes = int(self._L.acb_image_bytes(self._h))
            host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            _check(self._L.acb_image_write(self._h, host.data_ptr(), nbytes))
            img = host.to(torch.device("cuda", idx), non_blocking=False)
            self._images[idx] = img
        return img

    # ---- the sieve image (position-parallel scan: Bloom filter in shared memory + reverse trie in HBM/L2) ----
    ENGINE = __import__("os").environ.get("ACB200_ENGINE", "auto")   # "auto" | "sieve" | "table": kernel family (see scan_device)
    AUTO_PROFILE_BYTES = 4 << 20     # "auto": inputs below this never pay for the profiling pass
    SIEVE_SMEM_RESERVE = int(__import__("os").environ.get("ACB200_SIEVE_RESERVE_KB", "46")) * 1024   # 24 warps x (one ring slot of text + two queues); barrier
    SIEVE_W_MAX = 0                  # 0 = the builder chooses the primary window

    @staticmethod
    def _smem_optin(idx):
        props = _torch().cuda.get_device_properties(idx)
        return int(getattr(props, "shared_memory_per_block_optin", 227 * 1024))

    def sieve(self, device):
        """(device tensor, SieveDesc) of the sieve image on `device`, built and uploaded once."""
        torch = _require_cuda()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        ent = self._sieves.get(idx)
        if ent is None:
            smem = self._smem_optin(idx)
            nbytes = int(self._L.acb_sieve_build(self._h, max(4096, smem - self.SIEVE_SMEM_RESERVE), self.SIEVE_W_MAX))
            if nbytes == 0:
                raise RuntimeError(_capi.last_error())
            host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            _check(self._L.acb_sieve_write(self._h, host.data_ptr(), nbytes))
            desc = _capi.SieveDesc()
            _check(self._L.acb_sieve_describe(host.data_ptr(), C.byref(desc)))
            ent = (host.to(torch.device("cuda", idx)), desc)
            self._sieves[idx] = ent
        return ent

    def completions(self, device):
        """(device tensor, CompletionsDesc) of the completions image on `device` (csrc/completions.h: the reverse trie
        over every pattern's p[:-1] in token ids), built on the first call and uploaded once per device.  ValueError
        when the patterns are not in the token format."""
        torch = _require_cuda()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        with self._lock:
            ent = self._completions.get(idx)
            if ent is None:
                nbytes = C.c_uint64(0)
                if self._L.acb_completions_build(self._h, C.byref(nbytes)) != _capi.ACB_OK:
                    raise ValueError(_capi.last_error())
                host = torch.empty(nbytes.value, dtype=torch.uint8)
                _check(self._L.acb_completions_write(self._h, host.data_ptr(), nbytes.value))
                desc = _capi.CompletionsDesc()
                _check(self._L.acb_completions_describe(host.data_ptr(), C.byref(desc)))
                ent = (host.to(torch.device("cuda", idx)), desc)
                self._completions[idx] = ent
        return ent

    def sieve_geometry(self, device, task_bytes):
        """What shapes a sieve scan on `device` (for last_stats): the image's primary window, filter depth, probes and
        filter bytes, the ring depth the kernel runs with (acb_sieve_ring: the calling thread's tuning applies) and the
        task size.  None of it changes results; tests check it to know that an input reached the geometry it was made
        for."""
        torch = _torch()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        desc = self.sieve(device)[1]
        return {"window": desc.window, "last_level": desc.last_level, "probes": desc.probes, "bloom_bytes": desc.bloom_bytes,
                "ring": int(self._L.acb_sieve_ring(desc.bloom_bytes, self._smem_optin(idx))), "task_bytes": int(task_bytes)}

    # ---- the hot image (rows kept in shared memory), chosen from a sample of the data ----
    HOT_TABLE_BYTES = 40 * 1024   # with 32 warps of staging buffers next to it, this is what fits on chip
    HOT_COVERAGE_MIN = 0.99       # share of sampled state visits the hot rows must cover for the shared-memory kernel to be used

    def _max_hot_rows(self):
        return max(2, min(4096, self.HOT_TABLE_BYTES // (2 * self.num_columns) - 1))

    def _upload_hot(self, idx, visits_host):
        torch = _torch()
        rows = self._max_hot_rows()
        nbytes = int(self._L.acb_hot_bytes(self._h, rows))
        host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        vp = visits_host.ctypes.data if visits_host is not None else None
        _check(self._L.acb_hot_build(self._h, vp, rows, host.data_ptr(), nbytes))
        desc = _capi.HotDesc()
        _check(self._L.acb_hot_describe(host.data_ptr(), C.byref(desc)))
        return host.to(torch.device("cuda", idx)), desc

    def hot(self, device, data=None, offsets=None, overlapping=False):
        """The hot image on `device`.  Built from a profile of (data, offsets) the
        first time this automaton scans on the device, and again -- with
        exponential back-off -- when the kernel reports that the fast path keeps
        falling out of the hot set (the data changed character)."""
        torch = _torch()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        st = self._hot.get(idx)
        need = st is None or st["reprofile"]
        if need and data is not None and data.numel() > 0 and offsets is not None and offsets.numel() > 1:
            img = self.image(device)
            visits = torch.empty(self.num_states, dtype=torch.int32, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream
            n = offsets.numel() - 1
            _check(self._L.acb_profile(self._h, img.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                                       int(bool(overlapping)), visits.data_ptr(), stream))
            vh = visits.cpu().numpy().view(np.uint32)
            t, rows = self._upload_hot(idx, vh)
            # How much of the sampled scan the hot rows cover.  Every byte outside them costs the staged kernel a
            # detour through the exact scanner while 31 lanes wait; below ~99 % the segment kernel that reads the
            # table from global memory / L2 is faster (dense automata on random text: BASELINE configs 4 and 5).
            total_visits = int(vh.sum(dtype=np.uint64))
            if total_visits > 0 and rows.rows < self.num_states:
                top = np.partition(vh, len(vh) - rows.rows)[len(vh) - rows.rows:]
                coverage = float(top.sum(dtype=np.uint64)) / total_visits
            else:
                coverage = 1.0
            rows.reserved = 1 if coverage < self.HOT_COVERAGE_MIN else 0
            backoff = (st["backoff"] * 2) if st else 1
            st = {"tensor": t, "rows": rows, "reprofile": False, "calls": 0, "backoff": backoff, "coverage": coverage}
            self._hot[idx] = st
        elif st is None:
            t, rows = self._upload_hot(idx, None)
            st = {"tensor": t, "rows": rows, "reprofile": True, "calls": 0, "backoff": 1, "coverage": 1.0}
            self._hot[idx] = st
        return st

    def _note_trap_stats(self, st, groups: int, traps: int):
        st["calls"] += 1
        if st["rows"].reserved & 1:
            return  # scanning from global memory: the hot rows are not in use
        if groups > 4096 and traps * 10 > groups and st["calls"] >= st["backoff"]:
            st["reprofile"] = True
            st["calls"] = 0

    def _plan(self, data, n_haystacks: int):
        plan = _capi.Plan()
        _check(self._L.acb_plan_scan(self._h, data.data_ptr(), data.numel(), n_haystacks, C.byref(plan)))
        return plan

    @staticmethod
    def _ws_key(device, slot):
        return (device.index if device.index is not None else _torch().cuda.current_device(), slot)

    def _workspace(self, device, plan, n_haystacks: int, capacity: int, slot: int = 0):
        """Workspace `slot` on `device` (the host pipeline alternates between two), grown to fit, after making the
        current stream wait for the last reader of the views it handed out (_mark_read)."""
        torch = _torch()
        key = self._ws_key(device, slot)
        ws = self._ws.get(key)
        need = (ws is None or ws["n_units"] < plan.n_units or ws["n_segments"] < plan.n_segments or
                ws["scratch"].numel() < plan.scratch_words or ws["n_haystacks"] < n_haystacks or ws["capacity"] < capacity)
        if need:
            if ws is not None and ws.get("reader") is not None:
                ws["reader"].synchronize()   # an any_device comparison still reading the buffers about to be freed
            n_units = max(plan.n_units, ws["n_units"] if ws else 0, 1)
            n_seg = max(plan.n_segments, ws["n_segments"] if ws else 0, 1)
            n_hay = max(n_haystacks, ws["n_haystacks"] if ws else 0, 1)
            n_scr = max(plan.scratch_words, ws["scratch"].numel() if ws else 0, 16)
            cap = max(capacity, ws["capacity"] if ws else 0, 1024)
            dev = torch.device("cuda", key[0])
            ws = {
                "n_units": n_units, "n_segments": n_seg, "n_haystacks": n_hay, "capacity": cap,
                "raw": torch.empty((cap, 4), dtype=torch.int32, device=dev),
                "raw_seq": torch.empty(cap, dtype=torch.int32, device=dev),
                "raw_unit": torch.empty(cap, dtype=torch.int32, device=dev),
                "raw_aux": torch.empty(cap, dtype=torch.int32, device=dev),
                "unit_counts": torch.empty(n_units, dtype=torch.int32, device=dev),
                "unit_offsets": torch.empty(n_units + 1, dtype=torch.int64, device=dev),
                "seg_info": torch.empty((n_seg, 8), dtype=torch.int32, device=dev),
                "scratch": torch.zeros(n_scr, dtype=torch.int64, device=dev),  # zeroed: its head holds the kernels' counters
                "total": torch.zeros(8, dtype=torch.int64, device=dev),
                "out": torch.empty((cap, 4), dtype=torch.int32, device=dev),
                "match_offsets": torch.empty(n_hay + 1, dtype=torch.int64, device=dev),
            }
            self._ws[key] = ws
        reader = ws.pop("reader", None)
        if reader is not None:   # a comparison of an earlier call (maybe on another stream) reads this workspace first
            torch.cuda.current_stream(device).wait_event(reader)
        return ws

    def _mark_read(self, device, slot=0):
        """Records, on the current stream, that the views of workspace `slot` a scan handed out are read up to here:
        the next scan that uses the slot waits for this point (_workspace), on whatever stream or thread it runs."""
        torch = _torch()
        ws = self._ws.get(self._ws_key(device, slot))
        if ws is not None:
            reader = torch.cuda.Event()
            reader.record(torch.cuda.current_stream(device))
            ws["reader"] = reader

    def _list_attempt(self, device, plan, n_haystacks: int, capacity: Optional[int], launch, slot=0):
        """One list scan into workspace `slot`, with room for `capacity` records (None: max(1024, 2n)):
        launch(plan_ref, ws_struct_ref) -> rc calls the library.  A failure raises (ValueError for an unsupported
        request) with the workspace's counters zeroed.  -> the workspace; its "total" words say whether the list fit."""
        ws = self._workspace(device, plan, n_haystacks, capacity or max(1024, n_haystacks * 2), slot)
        rc = launch(C.byref(plan), C.byref(self._ws_struct(ws)))
        if rc != _capi.ACB_OK:
            err = _capi.last_error()
            ws["scratch"][:8].zero_()   # a scan that failed half way may have left its counters dirty
            raise (ValueError if rc == _capi.ACB_EUNSUPPORTED else RuntimeError)(err)
        return ws

    def _list_scan(self, device, plan, n_haystacks: int, capacity: Optional[int], launch):
        """_list_attempt on workspace slot 0 until the list fit (or was empty), each retry with room for all of it (a
        call whose list did not fit added nothing to its outputs) -> (workspace, its "total" words as a list)."""
        while True:
            ws = self._list_attempt(device, plan, n_haystacks, capacity, launch)
            tot = ws["total"].tolist()
            total, complete, raw_total = tot[0], tot[1], tot[4]
            if complete or (total == 0 and raw_total == 0):
                return ws, tot
            capacity = max(total, raw_total) + max(total, raw_total) // 8 + 16

    def _ws_struct(self, ws):
        s = _capi.Workspace()
        s.dev_raw = ws["raw"].data_ptr()
        s.dev_raw_seq = ws["raw_seq"].data_ptr()
        s.dev_raw_unit = ws["raw_unit"].data_ptr()
        s.dev_raw_aux = ws["raw_aux"].data_ptr()
        s.raw_capacity = ws["capacity"]
        s.dev_unit_counts = ws["unit_counts"].data_ptr()
        s.dev_unit_offsets = ws["unit_offsets"].data_ptr()
        s.dev_seg_info = ws["seg_info"].data_ptr()
        s.dev_scratch = ws["scratch"].data_ptr()
        s.dev_total = ws["total"].data_ptr()
        s.dev_out = ws["out"].data_ptr()
        s.out_capacity = ws["capacity"]
        s.dev_match_offsets = ws["match_offsets"].data_ptr()
        return s

    def check_overlapping(self, overlapping):
        # reference: the iterator is refused before any byte is read (src/lib.rs:52-54, 36-39)
        if overlapping and overlapping != 2 and self.matchkind != MatchKind.Standard:
            raise ValueError(f"match kind {self.matchkind.name} does not support overlapping searches")

    # ---- scans ------------------------------------------------------------------
    def _pick_engine(self, dev, data, offsets, overlapping):
        """Which kernel family scans (data, offsets): None = the sieve, else the hot image the table walkers use.
        Called under self._lock.  Results are identical; only speed and the device images a scan needs differ.
          table  the automaton walkers: best when the scan lives in a few hundred states that fit in shared memory
                 (sparse matches in text) -- the profile of the data says so (hot-row coverage);
          sieve  the position-parallel filter + exact verification: everything else (dense pattern sets, whose
                 states live in L2), and small inputs, where the profiling pass would cost more than the scan.
        The tuning knob's forced kernel and ENGINE override the profile."""
        torch = _torch()
        forced = _capi.current_kernel()
        if overlapping == 2 or forced == 5 or (forced == 0 and self.ENGINE == "sieve"):
            return None
        if forced in (1, 2, 3, 4) or self.ENGINE == "table":
            return self.hot(dev, data, offsets, overlapping)
        if self.implementation in (Implementation.ContiguousNFA, Implementation.NoncontiguousNFA):
            return None   # the caller asked for a compact (non-DFA) table format: that is the sieve image
        if data.numel() < self.AUTO_PROFILE_BYTES and self._hot.get(dev.index if dev.index is not None else torch.cuda.current_device()) is None:
            return None
        hot = self.hot(dev, data, offsets, overlapping)
        return None if hot["rows"].reserved & 1 else hot

    def any_device(self, data, offsets, out=None, sync: bool = True, flt=None):
        """Which haystacks of a device-resident batch contain an occurrence of any pattern -> bool CUDA tensor (n,).
        The answer does not depend on the match kind.  `out` (bool, (n,), contiguous, on the data's device): the
        answer is OR-ed into it, and haystacks already True there are not scanned.  With sync=False a call that runs
        the sieve returns right after enqueueing (and last_stats are not updated).

        Where the engine rule of scan_device picks the sieve, its kernel runs in the any-match mode (acb_any_match:
        no match list, work stops per haystack at its first match); where it picks a table walker (text whose scan
        stays in a few hot states), the walker's full scan is faster than the sieve's and its per-haystack counts give
        the answer.  That path always waits for its scan, whatever `sync` says: a match list that did not fit the
        workspace is only known on the host, and is scanned again with room for all of it (a truncated list would
        report haystacks with matches as False).  The next scan that reuses the workspace waits, on the device, for
        the comparison that reads it, so the returned tensor is the caller's own on either path, whatever stream or
        thread scans next."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        if out is not None and (out.dtype != torch.bool or out.dim() != 1 or out.numel() != max(n, 0) or out.device != dev or
                                not out.is_contiguous()):
            raise ValueError(f"out must be a contiguous bool tensor of shape ({max(n, 0)},) on {dev}")
        if n <= 0 or data.numel() == 0:
            return out if out is not None else torch.zeros(max(n, 0), dtype=torch.bool, device=dev)
        if data.numel() > self.WINDOW_BYTES:
            if not sync:
                raise ValueError(f"buffers above {self.WINDOW_BYTES} bytes are scanned in windows: sync=False is not available")
            return self._any_device_windows(data, offsets, out if out is not None else torch.zeros(n, dtype=torch.bool, device=dev), flt)
        with self._lock, torch.cuda.device(dev):
            use_sieve = flt is not None or self._pick_engine(dev, data, offsets, False) is None
            if use_sieve:
                if out is None:
                    out = torch.zeros(n, dtype=torch.bool, device=dev)
                sieve_t, _ = self.sieve(dev)
                plan = self._plan(data, n)
                scratch = torch.empty(3, dtype=torch.int64, device=dev)
                _check(self._L.acb_any_match_filtered(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                                                      out.data_ptr(), scratch.data_ptr(), _filter_struct(flt),
                                                      torch.cuda.current_stream(dev).cuda_stream))
            else:
                # scan_device (it takes the lock again and makes the same choice) with sync=True: it retries until the
                # list is complete.  Its match_offsets are a view of workspace slot 0, which every scan of this
                # automaton shares: the next scan that uses the slot waits for the event recorded after the comparison
                # (on whatever stream it runs), and a slot that grows first waits for it on the host.
                _, mo, _ = self.scan_device(data, offsets, False, False)
                hit = mo[1:] > mo[:-1]
                if out is None:
                    out = hit
                else:
                    out |= hit
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "any"}
                return out
        if sync:
            _, skipped, windows = scratch.tolist()
            task_bytes = int(plan.task_bytes)
            tasks = (data.numel() + (data.data_ptr() & 511) + task_bytes - 1) // task_bytes
            self.last_stats = {"engine": "sieve", "mode": "any", **self.sieve_geometry(dev, task_bytes), "tasks": tasks,
                               "tasks_skipped": skipped, "windows_skipped": windows, **self._set_stats(flt)}
        return out

    def _set_stats(self, flt):
        """last_stats entries of a call with pattern sets (none without)."""
        return {} if flt is None else {"pattern_sets": flt[0].n_sets}

    def _any_device_windows(self, data, offsets, out, flt=None):
        """any_device for buffers above WINDOW_BYTES: runs of whole haystacks that fit one call each get their slice
        of `out`; one haystack above the limit is scanned in windows that share max_pattern_len - 1 bytes (an
        occurrence lies inside one of them whole) and share its flag, stopping at the first window that sets it."""
        torch = _require_cuda()
        halo = max(self.max_pattern_len - 1, 0)
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if not large:
                self.any_device(data[start:end], offsets[h:h1 + 1] - start, out[h:h1], flt=_filter_slice(flt, h, h1))
                continue
            flag = out[h:h1]
            for w0, w1 in _windows(end - start, self.WINDOW_BYTES, halo):
                if bool(flag.item()):
                    break
                self.any_device(data[start + w0:start + w1], torch.tensor([0, w1 - w0], dtype=torch.int64, device=data.device), flag,
                                flt=_filter_slice(flt, h, h1))
        return out

    # ---- the first match per haystack (the crate's AhoCorasick::find) ---------------------------------------------
    def first_order(self, row):
        """Sort key of a (pattern, start, end) row: the first match of a haystack is the minimum over its overlapping
        matches (select_non_overlapping in csrc/capi.cu, first iteration)."""
        p, s, e = row
        if self.matchkind == MatchKind.Standard:
            return (e, s, p)
        if self.matchkind == MatchKind.LeftmostFirst:
            return (s, p)
        return (s, -e, p)

    def first_keys(self, data, offsets, keys, flt=None):
        """acb_find_first on the sieve: lowers the u64 keys (an int64 CUDA tensor (n,), -1 = no match yet) of a batch
        below WINDOW_BYTES; returns the u64[3] scratch tensor (task counter, tasks skipped, windows not scanned)."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        sieve_t, _ = self.sieve(dev)
        scratch = torch.empty(3, dtype=torch.int64, device=dev)
        _check(self._L.acb_find_first_filtered(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                                               keys.data_ptr(), scratch.data_ptr(), _filter_struct(flt), torch.cuda.current_stream(dev).cuda_stream))
        return scratch

    def first_rows(self, data, offsets, keys, flt=None):
        """acb_first_rows: keys -> int64 (n, 3) rows (pattern, start, end) in bytes, -1 rows where there is no match."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        sieve_t, _ = self.sieve(dev)
        rows = torch.empty((n, 3), dtype=torch.int64, device=dev)
        _check(self._L.acb_first_rows_filtered(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, keys.data_ptr(),
                                               rows.data_ptr(), _filter_struct(flt), torch.cuda.current_stream(dev).cuda_stream))
        return rows

    def _rows_to_codepoints(self, data, offsets, rows):
        torch = _torch()
        out = torch.empty_like(rows)
        _check(self._L.acb_rows_to_codepoints(data.data_ptr(), offsets.data_ptr(), offsets.numel() - 1, data.numel(), rows.data_ptr(),
                                              out.data_ptr(), torch.cuda.current_stream(data.device).cuda_stream))
        return out

    def first_device(self, data, offsets, codepoints: bool = False, flt=None):
        """Each haystack's first match for the match kind -> int64 CUDA tensor (n, 3) = (pattern, start, end), a row of
        -1 where a haystack has none; code point indexes with codepoints.  Row h is element 0 of haystack h's
        non-overlapping list (scan_device), for every match kind.

        Where the engine rule of scan_device picks the sieve, its kernel runs in the first-match mode (acb_find_first:
        no match list, work stops per haystack once no later position can beat the best match found), and the call
        returns without waiting for the device.  Where it picks a table walker, the rows come from the walker's full
        scan (which waits for it, as any_device's does), gathered on the device; the next scan that reuses the
        workspace waits for that gather."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        if n <= 0:
            return torch.empty((0, 3), dtype=torch.int64, device=dev)
        if data.numel() == 0:
            return torch.full((n, 3), -1, dtype=torch.int64, device=dev)
        if data.numel() > self.WINDOW_BYTES:
            rows = self._first_device_windows(data, offsets, flt)
            return self._rows_to_codepoints(data, offsets, rows) if codepoints else rows
        with self._lock, torch.cuda.device(dev):
            if flt is None and self._pick_engine(dev, data, offsets, False) is not None:
                m, mo, total = self.scan_device(data, offsets, False, codepoints)
                rows = torch.full((n, 3), -1, dtype=torch.int64, device=dev)
                if total:
                    has = mo[1:] > mo[:-1]
                    first = m[mo[:-1].clamp(max=total - 1), 1:4].to(torch.int64)
                    rows = torch.where(has[:, None], first, rows)
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "first"}
                return rows
            keys = torch.full((n,), -1, dtype=torch.int64, device=dev)   # all ones: no match yet
            scratch = self.first_keys(data, offsets, keys, flt)
            rows = self.first_rows(data, offsets, keys, flt)
            task_bytes = int(self._plan(data, n).task_bytes)
            self.last_stats = {"engine": "sieve", "mode": "first", **self.sieve_geometry(dev, task_bytes), **self._set_stats(flt),
                               "tasks": (data.numel() + (data.data_ptr() & 511) + task_bytes - 1) // task_bytes,
                               "skip_counters": scratch}   # device tensor: [task counter, tasks skipped, windows not scanned]
        return self._rows_to_codepoints(data, offsets, rows) if codepoints else rows

    def _first_device_windows(self, data, offsets, flt=None):
        """first_device (bytes) for buffers above WINDOW_BYTES: runs of whole haystacks that fit one call each get
        their rows (positions are haystack-relative: nothing to rebase); one haystack above the limit goes to
        _first_one_large."""
        torch = _require_cuda()
        dev = data.device
        rows = torch.full((offsets.numel() - 1, 3), -1, dtype=torch.int64, device=dev)
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                best = self._first_one_large(data[start:end], _filter_slice(flt, h, h1))
                if best is not None:
                    rows[h] = torch.tensor(best, dtype=torch.int64, device=dev)
            else:
                rows[h:h1] = self.first_device(data[start:end], offsets[h:h1 + 1] - start, flt=_filter_slice(flt, h, h1))
        return rows

    def _first_one_large(self, hay, flt=None):
        """The first match (pattern, start, end) in bytes, or None, of one haystack above WINDOW_BYTES, scanned in
        windows that share max_pattern_len - 1 bytes, in order.  A window sees every match that ends inside it and does
        not end inside the bytes it shares with its predecessor.  Standard: the first window with a match holds the
        earliest end.  The leftmost kinds: every match not seen yet ends past the current window, so it starts at or
        after the next window's start; the search stops once the best start lies strictly before that."""
        torch = _require_cuda()
        halo = max(self.max_pattern_len - 1, 0)
        best = None
        for w0, w1 in _windows(hay.numel(), self.WINDOW_BYTES, halo):
            p, s, e = self.first_device(hay[w0:w1], torch.tensor([0, w1 - w0], dtype=torch.int64, device=hay.device), flt=flt)[0].tolist()
            if p >= 0 and (best is None or self.first_order((p, s + w0, e + w0)) < self.first_order(best)):
                best = (p, s + w0, e + w0)
            if best is not None and (self.matchkind == MatchKind.Standard or best[1] < w1 - halo):
                break
        return best

    @contextlib.contextmanager
    def _host_staged(self, chunks):
        """Host buffers (bytes-like objects, one per haystack) -> (data, offsets) on the current device: gathered into
        the pinned staging buffer (_pack_host) and sent in one copy.  Also yields the host offsets and the host view of
        the bytes (valid inside the block).  Holds _host_lock: the staging buffer, and the workspaces until the results
        are on the host."""
        torch = _torch()
        dev = torch.device("cuda", torch.cuda.current_device())
        with self._host_lock:
            offs, head, total_bytes = _pack_host(lambda nbytes: self._pinned(nbytes).numpy(), chunks)
            host = self._pinned(head + total_bytes)
            d = host[:head + total_bytes].to(dev, non_blocking=True)
            yield d[head:], d[:8 * len(offs)].view(torch.int64), offs, host.numpy()[head:head + total_bytes]

    def first_host_batch(self, chunks: Sequence[bytes], codepoints: bool, patterns=None):
        """Host buffers (bytes-like objects, one per haystack) -> list of (pattern, start, end) or None: each one's first
        match.  The offsets and the haystacks go to the device in one copy (_host_staged); the rows come back in one."""
        _require_cuda()
        if len(chunks) == 0:
            return []
        with self._host_staged(chunks) as (data, offsets, _, _):
            flt = _host_sets(self, patterns, len(chunks), data.device) if patterns is not None else None
            rows = self.first_device(data, offsets, codepoints, flt).cpu().tolist()
        return [tuple(r) if r[0] >= 0 else None for r in rows]

    def any_host_batch(self, chunks: Sequence[bytes], patterns=None):
        """Host buffers (bytes-like objects, one per haystack) -> list of bool: does each contain any pattern.  The
        offsets and the haystacks go to the device in one copy (_host_staged)."""
        _require_cuda()
        if len(chunks) == 0:
            return []
        with self._host_staged(chunks) as (data, offsets, _, _):
            flt = _host_sets(self, patterns, len(chunks), data.device) if patterns is not None else None
            return self.any_device(data, offsets, flt=flt).cpu().tolist()

    # ---- match counts per haystack: len(find_matches_as_indexes(h, overlapping)) without the list ----------------
    def count_device(self, data, offsets, overlapping=False, capacity: Optional[int] = None, flt=None):
        """How many matches each haystack of a device-resident batch has -> int64 CUDA tensor (n,): the length of
        its list in scan_device, for every match kind.  Counts are the same in bytes and in code points, so no code
        point work is ever done.  An overlapping search on a leftmost automaton raises ValueError, as scan_device does.

        Where the engine rule of scan_device picks the sieve: an overlapping count is the sieve kernel's count mode
        (acb_count_overlapping: no list, no epilogue) and returns without waiting for the device; a non-overlapping
        count is the sieve's list scan and a count epilogue (acb_count_non_overlapping: the selection is counted, not
        packed; long per-haystack lists are counted by the whole grid), which waits for the device and scans again with
        more room when the list did not fit the workspace, as scan_device does.  Where the rule picks a table walker,
        the counts are diff(match_offsets) of its full scan, which waits for it; the next scan that reuses the
        workspace waits for that difference.  `capacity`: the workspace's first size, in records, as for scan_device."""
        self.check_overlapping(overlapping)
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        if n <= 0 or data.numel() == 0:
            return torch.zeros(max(n, 0), dtype=torch.int64, device=dev)
        if data.numel() > self.WINDOW_BYTES:
            return self._count_device_windows(data, offsets, overlapping, flt)
        with self._lock, torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            if flt is None and self._pick_engine(dev, data, offsets, overlapping) is not None:
                _, mo, _ = self.scan_device(data, offsets, overlapping, False)
                counts = mo[1:] - mo[:-1]
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "count", "long_stretches": 0}
                return counts
            sieve_t, _ = self.sieve(dev)
            counts = torch.zeros(n, dtype=torch.int64, device=dev)
            if overlapping:
                scratch = torch.empty(3, dtype=torch.int64, device=dev)
                _check(self._L.acb_count_overlapping_filtered(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n,
                                                              data.numel(), counts.data_ptr(), scratch.data_ptr(), _filter_struct(flt),
                                                              stream.cuda_stream))
                self.last_stats = {"engine": "sieve", "mode": "count", **self.sieve_geometry(dev, self._plan(data, n).task_bytes),
                                   "long_stretches": 0, **self._set_stats(flt)}
                return counts
            plan = self._plan(data, n)
            _, tot = self._list_scan(dev, plan, n, capacity, lambda plan_ref, ws_ref: self._L.acb_count_non_overlapping_filtered(
                self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(), plan_ref, ws_ref, counts.data_ptr(),
                _filter_struct(flt), stream.cuda_stream))
            long_stretches, raw_total = tot[2], tot[4]
            self.last_stats = {"engine": "sieve", "mode": "count", **self.sieve_geometry(dev, plan.task_bytes), "list_records": raw_total,
                               "long_stretches": long_stretches, **self._set_stats(flt)}
            return counts

    def _count_device_windows(self, data, offsets, overlapping, flt=None):
        """count_device for buffers above WINDOW_BYTES: runs of whole haystacks that fit one call each get their slice
        of the counts; one haystack above the limit goes to _count_one_large.  last_stats["long_stretches"] sums the
        runs'."""
        torch = _require_cuda()
        dev = data.device
        counts = torch.zeros(offsets.numel() - 1, dtype=torch.int64, device=dev)
        long_stretches, engine = 0, None
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                counts[h:h1] = self._count_one_large(data[start:end], overlapping, _filter_slice(flt, h, h1))
            else:
                counts[h:h1] = self.count_device(data[start:end], offsets[h:h1 + 1] - start, overlapping, flt=_filter_slice(flt, h, h1))
                long_stretches += self.last_stats.get("long_stretches", 0)
            engine = self.last_stats.get("engine") or engine
        torch.cuda.current_stream(dev).synchronize()
        self.last_stats = {"engine": engine, "mode": "count", "long_stretches": long_stretches, "windows": True, **self._set_stats(flt)}
        return counts

    def _count_one_large(self, hay, overlapping, flt=None):
        """The count (an int64 CUDA tensor (1,)) of one haystack above WINDOW_BYTES.
        Overlapping: windows that share max_pattern_len - 1 bytes (the head of each window but the first).  A window
        counts every match inside it; a match that lies wholly inside a window's head was counted by the window before,
        so the count of the head alone is subtracted.  Every other match ends past a head and starts inside its window.
        Non-overlapping: the overlapping rows of the windows, and acb_count_rows counts what the selection would pick."""
        torch = _require_cuda()
        dev = hay.device
        if overlapping:
            halo = max(self.max_pattern_len - 1, 0)
            total = torch.zeros(1, dtype=torch.int64, device=dev)
            for w0, w1 in _windows(hay.numel(), self.WINDOW_BYTES, halo):
                total += self.count_device(hay[w0:w1], torch.tensor([0, w1 - w0], dtype=torch.int64, device=dev), True, flt=flt)
                if w0 and halo:
                    total -= self.count_device(hay[w0:w0 + halo], torch.tensor([0, halo], dtype=torch.int64, device=dev), True, flt=flt)
            return total
        rows = self._overlapping_rows_large(hay, False, flt).contiguous()
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        if rows.shape[0]:
            scratch = torch.empty((rows.shape[0], 2), dtype=torch.int64, device=dev)   # 16 bytes per row
            _check(self._L.acb_count_rows(self._h, rows.data_ptr(), rows.shape[0], scratch.data_ptr(), count.data_ptr(),
                                          torch.cuda.current_stream(dev).cuda_stream))
        return count

    def count_host_batch(self, chunks: Sequence[bytes], overlapping, patterns=None):
        """Host buffers (bytes-like objects, one per haystack) -> list of int: each one's match count.  The offsets and
        the haystacks go to the device in one copy (_host_staged)."""
        _require_cuda()
        self.check_overlapping(overlapping)
        if len(chunks) == 0:
            return []
        with self._host_staged(chunks) as (data, offsets, _, _):
            flt = _host_sets(self, patterns, len(chunks), data.device) if patterns is not None else None
            return self.count_device(data, offsets, overlapping, flt=flt).cpu().tolist()

    # ---- match counts per pattern: bincount of find_matches_as_indexes' patterns, summed over a batch, without the list
    def pattern_counts_device(self, data, offsets, overlapping=False, capacity: Optional[int] = None):
        """How many matches each pattern has in a device-resident batch -> int64 CUDA tensor (n_patterns,): entry p is
        the number of records with pattern p in scan_device's list, summed over the haystacks.  Patterns with the same
        bytes keep their own ids.  An overlapping search on a leftmost automaton raises ValueError, as scan_device does.

        Where the engine rule of scan_device picks the sieve: an overlapping search is the sieve kernel's pattern mode
        (acb_pattern_counts_overlapping: no list, no epilogue) and returns without waiting for the device; a
        non-overlapping search is the sieve's list scan and a pattern epilogue (acb_pattern_counts_non_overlapping),
        which waits for the device and scans again with more room when the list did not fit (nothing was added then).
        Where the rule picks a table walker, the counts are the bincount of the pattern column of its full scan, which
        waits for it; the next scan that reuses the workspace waits for that bincount.  Batches above WINDOW_BYTES go
        in runs of whole haystacks, and one haystack above it in windows, all added into one tensor.  `capacity`: the
        workspace's first size, in records, as for scan_device."""
        self.check_overlapping(overlapping)
        torch = _require_cuda()
        counts = torch.zeros(self.n_patterns, dtype=torch.int64, device=data.device)
        n = offsets.numel() - 1
        if n <= 0 or data.numel() == 0:
            self.last_stats = {"engine": None, "mode": "pattern_counts", "long_stretches": 0}
            return counts
        if data.numel() > self.WINDOW_BYTES:
            self._pattern_counts_windows(counts, data, offsets, overlapping)
        else:
            self._pattern_counts_into(counts, data, offsets, overlapping, capacity)
        return counts

    def _pattern_counts_into(self, counts, data, offsets, overlapping, capacity=None):
        """Adds the per-pattern counts of a batch of at most WINDOW_BYTES to `counts`; sets last_stats."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        with self._lock, torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            if self._pick_engine(dev, data, offsets, overlapping) is not None:
                m, _, _ = self.scan_device(data, offsets, overlapping, False)
                counts += torch.bincount(m[:, 1].long(), minlength=self.n_patterns)
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "pattern_counts", "long_stretches": 0}
                return
            sieve_t, _ = self.sieve(dev)
            if overlapping:
                scratch = torch.empty(3, dtype=torch.int64, device=dev)
                _check(self._L.acb_pattern_counts_overlapping(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n,
                                                              data.numel(), counts.data_ptr(), scratch.data_ptr(), stream.cuda_stream))
                self.last_stats = {"engine": "sieve", "mode": "pattern_counts", **self.sieve_geometry(dev, self._plan(data, n).task_bytes),
                                   "long_stretches": 0}
                return
            plan = self._plan(data, n)
            _, tot = self._list_scan(dev, plan, n, capacity, lambda plan_ref, ws_ref: self._L.acb_pattern_counts_non_overlapping(
                self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(), plan_ref, ws_ref, counts.data_ptr(),
                stream.cuda_stream))
            long_stretches, raw_total = tot[2], tot[4]
            self.last_stats = {"engine": "sieve", "mode": "pattern_counts", **self.sieve_geometry(dev, plan.task_bytes),
                               "list_records": raw_total, "long_stretches": long_stretches}

    def _pattern_counts_windows(self, counts, data, offsets, overlapping):
        """pattern_counts_device above WINDOW_BYTES: runs of whole haystacks that fit one call each add their counts;
        one haystack above the limit goes to _pattern_counts_one_large.  last_stats["long_stretches"] sums the runs'."""
        torch = _require_cuda()
        long_stretches, engine = 0, None
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                self._pattern_counts_one_large(counts, data[start:end], overlapping)
            elif end > start:
                self._pattern_counts_into(counts, data[start:end], offsets[h:h1 + 1] - start, overlapping)
                long_stretches += self.last_stats.get("long_stretches", 0)
            engine = self.last_stats.get("engine") or engine
        torch.cuda.current_stream(data.device).synchronize()
        self.last_stats = {"engine": engine, "mode": "pattern_counts", "long_stretches": long_stretches, "windows": True}

    def _pattern_counts_one_large(self, counts, hay, overlapping):
        """Adds the per-pattern counts of one haystack above WINDOW_BYTES to `counts`.
        Overlapping: windows that share max_pattern_len - 1 bytes, as in _count_one_large.  A match wholly inside a
        window's head was counted by the window before, so the head's own counts are subtracted, pattern by pattern.
        Non-overlapping: the overlapping rows of the windows, the serial selection (acb_select_non_overlapping), and
        the bincount of the selected rows' patterns."""
        torch = _require_cuda()
        dev = hay.device
        if overlapping:
            halo = max(self.max_pattern_len - 1, 0)
            head = torch.zeros_like(counts)
            for w0, w1 in _windows(hay.numel(), self.WINDOW_BYTES, halo):
                self._pattern_counts_into(counts, hay[w0:w1], torch.tensor([0, w1 - w0], dtype=torch.int64, device=dev), True)
                if w0 and halo:
                    self._pattern_counts_into(head, hay[w0:w0 + halo], torch.tensor([0, halo], dtype=torch.int64, device=dev), True)
            counts -= head
            return
        rows = self._scan_one_large(hay, False, False)
        counts += torch.bincount(rows[:, 1], minlength=self.n_patterns)

    def pattern_counts_host_batch(self, chunks: Sequence[bytes], overlapping):
        """Host buffers (bytes-like objects, one per haystack) -> list of int: each pattern's match count over all of
        them.  The offsets and the haystacks go to the device in one copy (_host_staged)."""
        _require_cuda()
        self.check_overlapping(overlapping)
        if len(chunks) == 0:
            return [0] * self.n_patterns
        with self._host_staged(chunks) as (data, offsets, _, _):
            return self.pattern_counts_device(data, offsets, overlapping).cpu().tolist()

    # ---- hits per haystack: the distinct patterns of find_matches_as_indexes with their counts, without the list ----
    def hits_device(self, data, offsets, overlapping=False, capacity: Optional[int] = None):
        """Which patterns each haystack of a device-resident batch contains, and how often -> (row_offsets, patterns,
        counts), int64 CUDA tensors of shapes (n + 1,), (k,) and (k,): haystack h's hits are
        patterns[row_offsets[h]:row_offsets[h + 1]], ascending, each with how many records of its list in scan_device
        have that pattern.  torch.sparse_csr_tensor(row_offsets, patterns, counts, size=(n, n_patterns)) is the matrix:
        its row sums are count_device, its column sums pattern_counts_device.  The same in bytes and in code points.
        An overlapping search on a leftmost automaton raises ValueError, as scan_device does.

        Where the engine rule of scan_device picks the sieve: the sieve's list scan and a hits epilogue
        (acb_pattern_hits), which waits for the device and scans again with more room when the list or the counter rows
        did not fit.  Where the rule picks a table walker: torch.unique over haystack * n_patterns + pattern of its full
        scan, which waits for it; the next scan that reuses the workspace waits for that.  Batches above WINDOW_BYTES go
        in runs of whole haystacks; one haystack above it gets the nonzero entries of pattern_counts_device on it.
        `capacity`: the workspace's first size, in records, as for scan_device."""
        self.check_overlapping(overlapping)
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        if n <= 0 or data.numel() == 0:
            self.last_stats = {"engine": None, "mode": "matching_patterns", "long_stretches": 0, "rows": 0, "list_records": 0, "hits": 0}
            empty = torch.zeros(0, dtype=torch.int64, device=dev)
            return torch.zeros(max(n, 0) + 1, dtype=torch.int64, device=dev), empty, empty.clone()
        if data.numel() > self.WINDOW_BYTES:
            return self._hits_windows(data, offsets, overlapping)
        P = self.n_patterns
        with self._lock, torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            if self._pick_engine(dev, data, offsets, overlapping) is not None:
                m, _, _ = self.scan_device(data, offsets, overlapping, False)
                keys, counts = torch.unique(m[:, 0].long() * P + m[:, 1].long(), return_counts=True)
                row_offsets = torch.searchsorted(keys, torch.arange(n + 1, dtype=torch.int64, device=dev) * P)
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "matching_patterns", "long_stretches": 0,
                                   "rows": 0, "list_records": int(m.shape[0]), "hits": int(keys.numel())}
                return row_offsets, keys % P, counts
            sieve_t, _ = self.sieve(dev)
            plan = self._plan(data, n)
            cap = capacity
            row_words = self._hit_row_words
            rows = None
            while True:
                if row_words and (rows is None or rows.numel() < row_words):
                    rows = torch.empty(row_words, dtype=torch.int32, device=dev)
                ws = self._list_attempt(dev, plan, n, cap, lambda plan_ref, ws_ref: self._L.acb_pattern_hits(
                    self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(), int(bool(overlapping)), plan_ref,
                    ws_ref, rows.data_ptr() if rows is not None else None, row_words, stream.cuda_stream))
                hits, complete, long_stretches, n_rows, raw_total, need_words = ws["total"].tolist()[:6]
                if complete:
                    break
                if raw_total <= ws["capacity"] and need_words <= row_words:
                    raise RuntimeError("acb_pattern_hits reported an incomplete result with enough room")
                if raw_total > ws["capacity"]:
                    cap = raw_total + raw_total // 8 + 16
                row_words = max(row_words, need_words)
            self._hit_row_words = max(self._hit_row_words, need_words)   # (the next call with as many long stretches fits at once)
            row_offsets = ws["match_offsets"][: n + 1].clone()
            out = ws["out"][:hits]
            patterns, counts = out[:, 1].long(), out[:, 2].long()
            self._mark_read(dev)
            self.last_stats = {"engine": "sieve", "mode": "matching_patterns", **self.sieve_geometry(dev, plan.task_bytes),
                               "list_records": raw_total, "long_stretches": long_stretches, "rows": n_rows, "hits": hits}
            return row_offsets, patterns, counts

    def _hits_windows(self, data, offsets, overlapping):
        """hits_device for buffers above WINDOW_BYTES: runs of whole haystacks that fit one call each give their rows;
        one haystack above the limit gets the nonzero entries of pattern_counts_device (which windows it).  last_stats
        sums the runs'."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        sizes, patterns, counts = [], [], []
        stats = {"long_stretches": 0, "rows": 0, "list_records": 0}
        engine = None
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                pc = self.pattern_counts_device(data[start:end], torch.tensor([0, end - start], dtype=torch.int64, device=dev), overlapping)
                pids = torch.nonzero(pc).flatten()
                sizes.append(torch.tensor([pids.numel()], dtype=torch.int64, device=dev))
                patterns.append(pids)
                counts.append(pc[pids])
            else:
                ro, p, c = self.hits_device(data[start:end], offsets[h:h1 + 1] - start, overlapping)
                sizes.append(ro[1:] - ro[:-1])
                patterns.append(p)
                counts.append(c)
                for k in stats:
                    stats[k] += self.last_stats.get(k, 0)
            engine = self.last_stats.get("engine") or engine
        row_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.cat(sizes), 0, out=row_offsets[1:])
        patterns, counts = torch.cat(patterns), torch.cat(counts)
        self.last_stats = {"engine": engine, "mode": "matching_patterns", **stats, "hits": int(patterns.numel()), "windows": True}
        return row_offsets, patterns, counts

    def hits_host_batch(self, chunks: Sequence[bytes], overlapping):
        """Host buffers (bytes-like objects, one per haystack) -> one list per haystack: the distinct pattern ids of its
        matches, ascending.  The offsets and the haystacks go to the device in one copy (_host_staged)."""
        _require_cuda()
        self.check_overlapping(overlapping)
        n = len(chunks)
        if n == 0:
            return []
        with self._host_staged(chunks) as (data, offsets, _, _):
            ro, p, _ = self.hits_device(data, offsets, overlapping)
            ro, p = ro.cpu().tolist(), p.cpu().tolist()
        return [p[ro[i]:ro[i + 1]] for i in range(n)]

    # ---- match masks: which bytes lie inside a match of find_matches_as_indexes, without the list ----------------
    def mask_device(self, data, offsets, overlapping=False, capacity: Optional[int] = None, flt=None, words=None, bit_base: int = 0):
        """Which bytes of a device-resident batch lie inside one of its haystacks' matches -> the packed mask, an int32
        CUDA tensor of u32 words: bit p % 32 of word p // 32 = byte p of `data` is covered (start <= p - offsets[h] < end
        for a record of haystack h's list in scan_device).  With `words` given, the bits go to bit_base + p and are
        OR-ed into it (runs and windows share one mask).  An overlapping search on a leftmost automaton raises
        ValueError, as scan_device does.

        Where the engine rule of scan_device picks the sieve (always with pattern sets): an overlapping search is the
        sieve kernel's cover mode (acb_match_mask_overlapping: the longest match at each end position, no list) and
        returns without waiting for the device; a non-overlapping search is the sieve's list scan and a mask epilogue
        (acb_match_mask_non_overlapping), which waits for the device and scans again with more room when the list did
        not fit (nothing was OR-ed then).  Where the rule picks a table walker, the rows of its full scan are OR-ed in
        with acb_mask_rows; the next scan that reuses the workspace waits for that.  Batches above WINDOW_BYTES go in
        runs of whole haystacks, and one haystack above it in windows.  `capacity`: as for scan_device."""
        self.check_overlapping(overlapping)
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        if words is None:
            words = torch.zeros((data.numel() + 31) // 32, dtype=torch.int32, device=dev)
        if n <= 0 or data.numel() == 0:
            self.last_stats = {"engine": None, "mode": "match_mask", "long_stretches": 0, **self._set_stats(flt)}
            return words
        if data.numel() > self.WINDOW_BYTES:
            self._mask_windows(words, bit_base, data, offsets, overlapping, flt)
            return words
        with self._lock, torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            if flt is None and self._pick_engine(dev, data, offsets, overlapping) is not None:
                m, _, _ = self.scan_device(data, offsets, overlapping, False)
                self._mask_rows(words, bit_base, m, offsets)
                self._mark_read(dev)
                self.last_stats = {"engine": self.last_stats.get("engine", "table"), "mode": "match_mask", "long_stretches": 0}
                return words
            sieve_t, _ = self.sieve(dev)
            if overlapping:
                scratch = torch.empty(3, dtype=torch.int64, device=dev)
                _check(self._L.acb_match_mask_overlapping_filtered(self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n,
                                                                   data.numel(), words.data_ptr(), bit_base, scratch.data_ptr(),
                                                                   _filter_struct(flt), stream.cuda_stream))
                self.last_stats = {"engine": "sieve", "mode": "match_mask", **self.sieve_geometry(dev, self._plan(data, n).task_bytes),
                                   **self._set_stats(flt)}
                return words
            plan = self._plan(data, n)
            _, tot = self._list_scan(dev, plan, n, capacity, lambda plan_ref, ws_ref: self._L.acb_match_mask_non_overlapping_filtered(
                self._h, sieve_t.data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(), plan_ref, ws_ref, words.data_ptr(),
                bit_base, _filter_struct(flt), stream.cuda_stream))
            long_stretches, raw_total = tot[2], tot[4]
            self.last_stats = {"engine": "sieve", "mode": "match_mask", **self.sieve_geometry(dev, plan.task_bytes),
                               "list_records": raw_total, "long_stretches": long_stretches, **self._set_stats(flt)}
            return words

    def _mask_rows(self, words, bit_base: int, rows, offsets):
        """acb_mask_rows: OR the spans of selected rows (int32 acb_match records or int64 rows, haystack-relative) into
        `words` at bit_base + offsets[h] + [start, end)."""
        torch = _torch()
        if rows.shape[0] == 0:
            return
        rows = rows.contiguous()
        _check(self._L.acb_mask_rows(rows.data_ptr(), rows.element_size(), rows.shape[0], offsets.data_ptr(), offsets.numel() - 1,
                                     words.data_ptr(), bit_base, torch.cuda.current_stream(rows.device).cuda_stream))

    def _mask_windows(self, words, bit_base: int, data, offsets, overlapping, flt=None):
        """mask_device above WINDOW_BYTES: runs of whole haystacks that fit one call each OR their bits, from the run's
        first byte on; one haystack above the limit goes to _mask_one_large.  last_stats["long_stretches"] sums the
        runs'."""
        torch = _require_cuda()
        long_stretches, engine = 0, None
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                self._mask_one_large(words, bit_base + start, data[start:end], overlapping, _filter_slice(flt, h, h1))
            elif end > start:
                self.mask_device(data[start:end], offsets[h:h1 + 1] - start, overlapping, flt=_filter_slice(flt, h, h1), words=words,
                                 bit_base=bit_base + start)
                long_stretches += self.last_stats.get("long_stretches", 0)
            engine = self.last_stats.get("engine") or engine
        torch.cuda.current_stream(data.device).synchronize()
        self.last_stats = {"engine": engine, "mode": "match_mask", "long_stretches": long_stretches, "windows": True,
                           **self._set_stats(flt)}

    def _mask_one_large(self, words, bit_base: int, hay, overlapping, flt=None):
        """OR the mask of one haystack above WINDOW_BYTES into `words` from bit_base on.
        Overlapping: windows that share max_pattern_len - 1 bytes, each OR-ed at its own start.  Every match lies
        inside some window whole, and a match seen by two windows sets the same bits twice: nothing is subtracted.
        Non-overlapping: the selected rows of _scan_one_large, OR-ed with acb_mask_rows."""
        torch = _require_cuda()
        dev = hay.device
        if overlapping:
            for w0, w1 in _windows(hay.numel(), self.WINDOW_BYTES, max(self.max_pattern_len - 1, 0)):
                self.mask_device(hay[w0:w1], torch.tensor([0, w1 - w0], dtype=torch.int64, device=dev), True, flt=flt, words=words,
                                 bit_base=bit_base + w0)
            return
        rows = self._scan_one_large(hay, False, False, flt)
        self._mask_rows(words, bit_base, rows, torch.tensor([0, hay.numel()], dtype=torch.int64, device=dev))

    def unpack_mask(self, words, n: int, stride: int = 1):
        """acb_mask_unpack: bool CUDA tensor (n,), entry i = bit stride * i of the packed mask."""
        torch = _require_cuda()
        out = torch.empty(n, dtype=torch.bool, device=words.device)
        _check(self._L.acb_mask_unpack(words.data_ptr(), 0, stride, n, out.data_ptr(), torch.cuda.current_stream(words.device).cuda_stream))
        return out

    def spans_host_batch(self, chunks: Sequence[bytes], overlapping, codepoints: bool, patterns=None, unit: int = 1):
        """Host buffers (bytes-like objects, one per haystack) -> one list of (start, end) per haystack: the maximal
        runs of covered positions, haystack-relative, in code points with `codepoints`, else in bytes divided by `unit`.
        The offsets and the haystacks go to the device in one copy (_host_staged); the packed mask (one bit per byte)
        comes back."""
        _require_cuda()
        self.check_overlapping(overlapping)
        if len(chunks) == 0:
            return []
        with self._host_staged(chunks) as (data, offsets, offs, text):
            flt = _host_sets(self, patterns, len(chunks), data.device) if patterns is not None else None
            words = self.mask_device(data, offsets, overlapping, flt=flt).cpu().numpy()
            text = text.copy() if codepoints else None
        return spans_from_words(words, offs, text, unit)

    def scan_device(self, data, offsets, overlapping=False, codepoints=False, capacity: Optional[int] = None,
                    sync: bool = True, ws_slot: int = 0, flt=None):
        """Scan a device-resident batch.  data: uint8 CUDA tensor, offsets: int64
        CUDA tensor (n+1).  One haystack of any size is simply n = 1.  Returns
        (matches, match_offsets, total): matches is an int32 CUDA tensor
        (total, 4) = (haystack, pattern, start, end) in the reference's order,
        match_offsets (n+1) brackets each haystack's rows.  With sync=False the
        call returns right after enqueueing (total is the 8-entry device status
        tensor and matches the whole capacity-sized buffer).

        The returned tensors are VIEWS of this automaton's workspace `ws_slot` on the
        device: they are valid until the next scan that uses the same slot (copy them,
        or use scan_host / the find_* methods, when several threads share one automaton)."""
        torch = _require_cuda()
        self.check_overlapping(overlapping)
        dev = data.device
        n = offsets.numel() - 1
        if data.numel() > self.WINDOW_BYTES:
            if not sync:
                raise ValueError(f"buffers above {self.WINDOW_BYTES} bytes are scanned in windows: sync=False is not available")
            return self._scan_device_windows(data, offsets, overlapping, codepoints, flt)
        img = self.image(dev)
        cap = capacity
        stream = torch.cuda.current_stream(dev).cuda_stream
        with self._lock, torch.cuda.device(dev):
            hot = self._pick_engine(dev, data, offsets, overlapping) if flt is None else None   # (pattern sets: the sieve)
            use_sieve = hot is None
            if use_sieve:
                sieve_t, sieve_d = self.sieve(dev)
            plan = self._plan(data, n)
            while True:
                ws = self._list_attempt(dev, plan, n, cap, lambda plan_ref, ws_ref: self._L.acb_scan_batch_filtered(
                    self._h, img.data_ptr(), hot["tensor"].data_ptr() if hot else None, C.byref(hot["rows"]) if hot else None,
                    sieve_t.data_ptr() if use_sieve else None, data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                    2 if overlapping == 2 else int(bool(overlapping)), int(bool(codepoints)), plan_ref, ws_ref, _filter_struct(flt),
                    stream), ws_slot)
                if not sync:
                    return ws["out"], ws["match_offsets"][: n + 1], ws["total"]
                tot = ws["total"].tolist()
                total, complete, raw_total = tot[0], tot[1], tot[4]
                if hot:
                    self._note_trap_stats(hot, tot[2], tot[3])
                    self.last_stats = {"engine": "table", "groups": tot[2], "traps": tot[3], "repairs": tot[5], "segments": plan.n_segments,
                                       "paths": tot[6],
                                       "hot_rows": hot["rows"].rows, "hot_rows128": hot["rows"].rows128,
                                       "hot_visited": hot["rows"].visited, "hot_coverage": round(hot.get("coverage", 1.0), 5),
                                       "global_table": bool(hot["rows"].reserved & 1),
                                       "segment_bytes": plan.segment_bytes, "lane_stride": plan.lane_stride}
                else:
                    self.last_stats = {"engine": "sieve", **self.sieve_geometry(dev, plan.task_bytes), "nodes": sieve_d.nodes,
                                       "keys": sieve_d.keys, "filter_entries": sieve_d.filter_entries, "list_records": raw_total,
                                       **self._set_stats(flt)}
                if complete or (total == 0 and raw_total == 0):
                    return ws["out"][:total], ws["match_offsets"][: n + 1], total
                cap = max(total, raw_total) + max(total, raw_total) // 8 + 16

    # One kernel call addresses its buffer with 32-bit offsets.  Larger inputs are cut up here: a batch into
    # runs of whole haystacks, a single haystack above the limit into overlapping windows.
    WINDOW_BYTES = (1 << 31) - (1 << 16)   # (below 2^31: every offset of one call is a non-negative int32)

    def _scan_device_windows(self, data, offsets, overlapping, codepoints, flt=None):
        """scan_device for buffers above WINDOW_BYTES.  Same results, as int64 tensors
        (offsets no longer fit 32 bits): (matches (k, 4) int64, match_offsets (n + 1) int64, total).
        Everything stays on the device; the host only learns where the runs of whole haystacks end."""
        torch = _require_cuda()
        dev = data.device
        n = offsets.numel() - 1
        parts = []          # (k, 4) int64 tensors in haystack order
        mo = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        base_count = 0
        for h, h1, start, end, large in _haystack_runs(offsets, self.WINDOW_BYTES):
            if large:
                part = self._scan_one_large(data[start:end], overlapping, codepoints, _filter_slice(flt, h, h1))
                part[:, 0] = h
                parts.append(part)
                base_count += int(part.shape[0])
                mo[h + 1] = base_count
                continue
            sub_offs = offsets[h:h1 + 1] - start
            _t0 = __import__("time").perf_counter() if _TRACE else 0
            m, mo_run, total = self.scan_device(data[start:end], sub_offs, overlapping, codepoints, flt=_filter_slice(flt, h, h1))
            _t1 = __import__("time").perf_counter() if _TRACE else 0
            part = m.to(torch.int64)
            if h:
                part[:, 0] += h
            parts.append(part)
            mo[h + 1:h1 + 1] = mo_run[1:h1 - h + 1].to(torch.int64) + base_count
            base_count += int(total)
            if _TRACE:
                torch.cuda.synchronize()
                print(f"[trace] run haystacks {h}..{h1} ({end - start} B): scan_device {(_t1 - _t0) * 1e3:.2f} ms, post {(__import__('time').perf_counter() - _t1) * 1e3:.2f} ms, total {total}", flush=True)
        out = torch.cat(parts, dim=0) if len(parts) != 1 else parts[0]
        if not parts:
            out = torch.zeros((0, 4), dtype=torch.int64, device=dev)
        return out, mo, int(out.shape[0])

    def _scan_one_large(self, hay, overlapping, codepoints, flt=None):
        """One haystack above WINDOW_BYTES (BASELINE config 4: one 4 GiB haystack, overlapping).  The OVERLAPPING list
        is exact window by window: windows that share max_pattern_len - 1 bytes are independent (what ends at a position
        depends on no more than that), each keeps the matches that END beyond the shared bytes.  A non-overlapping
        search restarts at every match end, which chains the windows to each other: its result is SELECTED from the
        overlapping list afterwards (acb_select_non_overlapping; SURVEY.md 8c), for all three match kinds."""
        torch = _require_cuda()
        dev = hay.device
        rows = self._overlapping_rows_large(hay, codepoints, flt)
        if overlapping or rows.shape[0] == 0:
            return rows
        rows = rows.contiguous()
        out = torch.empty_like(rows)
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        _check(self._L.acb_select_non_overlapping(self._h, rows.data_ptr(), rows.shape[0], out.data_ptr(), count.data_ptr(),
                                                  torch.cuda.current_stream(dev).cuda_stream))
        return out[: int(count.item())]

    def _overlapping_rows_large(self, hay, codepoints, flt=None):
        """The overlapping list of one haystack above WINDOW_BYTES, whatever the match kind, as int64 rows (haystack,
        pattern, start, end) in the reference's order (see _scan_one_large)."""
        torch = _require_cuda()
        dev = hay.device

        def scan_window(window):
            one = torch.tensor([0, window.numel()], dtype=torch.int64, device=dev)
            m, _, _ = self._scan_overlapping_list(window, one, codepoints, flt)
            return m.to(torch.int64)

        parts = scan_in_windows(scan_window, hay, self.WINDOW_BYTES, max(self.max_pattern_len - 1, 0), codepoints)
        return torch.cat(parts, dim=0) if parts else torch.zeros((0, 4), dtype=torch.int64, device=dev)

    def _scan_overlapping_list(self, data, offsets, codepoints, flt=None):
        """The overlapping match list whatever the automaton's match kind: the sieve's structures do not depend on the
        kind (overlapping = 2 is the library-internal form of the request; the public overlapping=True on a leftmost
        automaton stays an error, like the reference's)."""
        return self.scan_device(data, offsets, 2, codepoints, flt=flt)

    # ---- host-resident input (the reference's situation: src/lib.rs:229-249, 422-434 take host str / buffers) ----
    HOST_CHUNK_BYTES = 1 << 30     # inputs up to this size go in one piece (the scan is ~100x faster than PCIe: nothing to hide);
                                   # larger ones in runs of this size: copy of run i+1 || scan of run i || results of run i-1
    _staging = None                # grow-only pinned staging buffer for inputs that are not pinned already

    def _pinned(self, nbytes: int):
        torch = _torch()
        st = self._staging
        if st is None or st.numel() < nbytes:
            st = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, pin_memory=True)
            self._staging = st
        return st

    def scan_host(self, data, offsets, overlapping: bool = False, codepoints: bool = False, chunk_bytes: Optional[int] = None):
        """Scan a batch that lives in HOST memory: data = 1-D uint8 (numpy array or CPU torch tensor; pinned memory
        makes the copies asynchronous), offsets = int64 (n + 1).  Returns host numpy arrays
        (matches (k, 4) uint32 -- int64 when a window path was needed --, match_offsets (n + 1) int64).

        Large inputs are cut into runs of whole haystacks of about `chunk_bytes`: the host->device copy of run i+1
        (copy stream, second device buffer) overlaps the scan of run i, whose results are copied back while run i+1
        is scanned (two workspaces).  The whole call holds the automaton's lock, so threads sharing one automaton
        are serialised here instead of corrupting each other's workspace."""
        torch = _require_cuda()
        self.check_overlapping(overlapping)
        if isinstance(data, np.ndarray):
            hdata = torch.from_numpy(data) if data.flags.writeable else torch.from_numpy(data.copy())
        else:
            hdata = data
        offs = offsets.numpy() if hasattr(offsets, "numpy") else np.asarray(offsets)
        offs = np.ascontiguousarray(offs, dtype=np.int64)
        n = len(offs) - 1
        total_bytes = int(offs[-1] - offs[0]) if n > 0 else 0
        dev = torch.device("cuda", torch.cuda.current_device())
        chunk = int(chunk_bytes or self.HOST_CHUNK_BYTES)
        chunk = min(chunk, self.WINDOW_BYTES)   # every run is one kernel call (scanned with sync=False: no window path)
        with self._host_lock:
            if n <= 0 or total_bytes <= chunk or int(np.max(np.diff(offs))) > self.WINDOW_BYTES:
                # one shot (small input), or the oversized-haystack window path
                lo, hi = (int(offs[0]), int(offs[-1])) if n > 0 else (0, 0)
                d_data = hdata[lo:hi].to(dev, non_blocking=True)
                d_offs = torch.from_numpy(offs - lo).to(dev, non_blocking=True)
                m, moffs, _ = self.scan_device(d_data, d_offs, overlapping, codepoints)
                m = m.cpu().numpy()
                return (m.view(np.uint32) if m.dtype == np.int32 else m), moffs.cpu().numpy().astype(np.int64)
            # runs of whole haystacks
            cuts = [0]
            while cuts[-1] < n:
                h0 = cuts[-1]
                h1 = int(np.searchsorted(offs, offs[h0] + chunk, side="right")) - 1
                cuts.append(min(max(h1, h0 + 1), n))
            runs = list(zip(cuts[:-1], cuts[1:]))
            max_bytes = max(int(offs[b] - offs[a]) for a, b in runs)
            max_hay = max(b - a for a, b in runs)
            dbuf = [torch.empty(max_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
            doff = [torch.empty(max_hay + 1, dtype=torch.int64, device=dev) for _ in range(2)]
            hoff = [torch.empty(max_hay + 1, dtype=torch.int64, pin_memory=True) for _ in range(2)]
            main = torch.cuda.current_stream(dev)
            copier = torch.cuda.Stream(device=dev)
            scanned = [None, None]
            parts, counts = [], np.zeros(n, dtype=np.int64)
            cap = max(4096, 2 * max_hay)

            def collect(job):
                slot, a, b, nbytes, out, mo, tot = job
                t = tot.tolist()            # waits for that run's scan only
                total, complete, raw_total = t[0], t[1], t[4]
                if not (complete or (total == 0 and raw_total == 0)):
                    # rare: the run had more matches than room; redo it with what it needs
                    m, mo2, total = self.scan_device(dbuf[slot][:nbytes], doff[slot][: b - a + 1], overlapping, codepoints,
                                                     capacity=max(total, raw_total) + max(total, raw_total) // 8 + 16, ws_slot=slot)
                    out, mo = m, mo2
                part = np.empty((total, 4), dtype=np.uint32)
                if total:
                    torch.from_numpy(part.view(np.int32)).copy_(out[:total])   # one D2H copy straight into the result array
                    if a:
                        part[:, 0] += a
                parts.append(part)
                run_mo = np.empty(b - a + 1, dtype=np.int64)
                torch.from_numpy(run_mo).copy_(mo[: b - a + 1])
                counts[a:b] = np.diff(run_mo)

            pending = None
            for i, (a, b) in enumerate(runs):
                slot = i & 1
                nbytes = int(offs[b] - offs[a])
                with torch.cuda.stream(copier):
                    if scanned[slot] is not None:
                        copier.wait_event(scanned[slot])   # the scan that read this device buffer two runs ago
                    dbuf[slot][:nbytes].copy_(hdata[int(offs[a]):int(offs[b])], non_blocking=True)
                    hoff[slot][: b - a + 1].copy_(torch.from_numpy(offs[a:b + 1] - offs[a]))
                    doff[slot][: b - a + 1].copy_(hoff[slot][: b - a + 1], non_blocking=True)
                    copied = torch.cuda.Event()
                    copied.record(copier)
                main.wait_event(copied)
                if pending is not None and pending[0] == slot:
                    collect(pending)        # (never: slots alternate) keeps the workspace of this slot free
                    pending = None
                out, mo, tot = self.scan_device(dbuf[slot][:nbytes], doff[slot][: b - a + 1], overlapping, codepoints,
                                                capacity=cap, sync=False, ws_slot=slot)
                ev = torch.cuda.Event()
                ev.record(main)
                scanned[slot] = ev
                job = (slot, a, b, nbytes, out, mo, tot)
                if pending is not None:
                    collect(pending)        # D2H of the previous run while this one is being scanned
                pending = job
            collect(pending)
            m = np.concatenate(parts, axis=0) if parts else np.zeros((0, 4), dtype=np.uint32)
            mo = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(counts, out=mo[1:])
            return m, mo

    # ---- one small haystack per call: the reference's own usage (benchmarks/test_comparison.py:119-122) ----
    SMALL_CALL_BYTES = 256 << 10   # up to here a single-haystack call takes the lean path below
    SMALL_CALL_ROWS = 64           # matches copied back with the status words in ONE transfer (more: a second copy)

    def _small_ctx(self, dev):
        """Everything a small call needs, allocated once per device: pinned and device input buffers (offsets first,
        then the bytes), a workspace whose status words and output rows are adjacent (one D2H copy fetches both), its
        ctypes description, the sieve image."""
        torch = _torch()
        idx = dev.index
        ctx = self._small.get(idx)
        if ctx is None:
            cap_b = self.SMALL_CALL_BYTES
            sieve_t, sieve_d = self.sieve(dev)
            img = self.image(dev)
            h_in = torch.zeros(16 + cap_b + 16, dtype=torch.uint8, pin_memory=True)
            d_in = torch.zeros(16 + cap_b + 16, dtype=torch.uint8, device=dev)
            plan = _capi.Plan()
            _check(self._L.acb_plan_scan(self._h, d_in.data_ptr() + 16, cap_b, 1, C.byref(plan)))
            cap = 4096
            n_units = int(plan.n_units) + 8
            res = torch.zeros(8 + 2 * cap, dtype=torch.int64, device=dev)
            ws = {
                "n_units": n_units, "n_segments": int(plan.n_segments) + 4, "n_haystacks": 1, "capacity": cap,
                "raw": torch.empty((cap, 4), dtype=torch.int32, device=dev),
                "raw_seq": torch.empty(cap, dtype=torch.int32, device=dev),
                "raw_unit": torch.empty(cap, dtype=torch.int32, device=dev),
                "raw_aux": torch.empty(cap, dtype=torch.int32, device=dev),
                "unit_counts": torch.empty(n_units, dtype=torch.int32, device=dev),
                "unit_offsets": torch.empty(n_units + 1, dtype=torch.int64, device=dev),
                "seg_info": torch.empty((int(plan.n_segments) + 4, 8), dtype=torch.int32, device=dev),
                "scratch": torch.zeros(int(plan.scratch_words) + 64, dtype=torch.int64, device=dev),
                "total": res[:8], "out": res[8:].view(torch.int32).view(cap, 4),
                "match_offsets": torch.empty(2, dtype=torch.int64, device=dev),
            }
            ctx = {"h_in": h_in, "d_in": d_in, "hv": h_in.numpy(), "res": res, "ws": ws, "st": self._ws_struct(ws),
                   "h_res": torch.zeros(8 + 2 * self.SMALL_CALL_ROWS, dtype=torch.int64, pin_memory=True),
                   "sieve": sieve_t, "img": img, "plan": plan, "max_scratch": int(plan.scratch_words) + 64, "max_units": n_units}
            ctx["hr"] = ctx["h_res"].numpy()
            self._small[idx] = ctx
        return ctx

    def _small_call(self, hay, overlapping: bool, codepoints: bool):
        """One haystack of at most SMALL_CALL_BYTES (a bytes-like object): one H2D copy, scan + epilogue, one D2H copy of
        (status, first rows), one synchronisation.  -> uint32 (k, 4) host array."""
        torch = _require_cuda()
        dev = torch.device("cuda", torch.cuda.current_device())
        n = len(hay)
        with self._host_lock:
            ctx = self._small_ctx(dev)
            hv = ctx["hv"]
            hv[:16].view(np.int64)[:] = (0, n)
            if n:
                hv[16:16 + n] = np.frombuffer(hay, dtype=np.uint8)
            d_in = ctx["d_in"]
            d_in[:16 + n].copy_(ctx["h_in"][:16 + n], non_blocking=True)
            plan = ctx["plan"]
            base = d_in.data_ptr()
            _check(self._L.acb_plan_scan(self._h, base + 16, n, 1, C.byref(plan)))
            if plan.scratch_words > ctx["max_scratch"] or plan.n_units > ctx["max_units"]:
                return None   # (a tuning knob changed the plan beyond what was allocated: let the general path do it)
            stream = torch.cuda.current_stream(dev)
            rc = self._L.acb_scan_batch(self._h, ctx["img"].data_ptr(), None, None, ctx["sieve"].data_ptr(), base + 16, base, 1, n,
                                        int(bool(overlapping)), int(bool(codepoints)), C.byref(plan), C.byref(ctx["st"]), stream.cuda_stream)
            if rc != _capi.ACB_OK:
                err = _capi.last_error()
                ctx["ws"]["scratch"][:8].zero_()   # a scan that failed half way may have left its counters dirty
                raise (ValueError if rc == _capi.ACB_EUNSUPPORTED else RuntimeError)(err)
            ctx["h_res"].copy_(ctx["res"][: ctx["h_res"].numel()], non_blocking=True)
            stream.synchronize()
            hr = ctx["hr"]
            total, complete = int(hr[0]), int(hr[1])
            if not complete:
                return None   # more matches than the small workspace holds: the general path sizes one
            if total <= self.SMALL_CALL_ROWS:
                return hr[8:8 + 2 * total].view(np.uint32).reshape(total, 4).copy()
            return ctx["ws"]["out"][:total].cpu().numpy().view(np.uint32)

    def scan_host_batch(self, chunks: Sequence[bytes], overlapping: bool, codepoints: bool, patterns=None):
        """Host buffers (bytes-like objects, one per haystack) in, host numpy out: (matches uint32 (k,4),
        match_offsets int64 (n+1)).  The haystacks are gathered into this automaton's pinned staging buffer
        (for a single haystack: one copy straight out of the caller's buffer), then scan_host takes over."""
        torch = _require_cuda()
        self.check_overlapping(overlapping)
        n = len(chunks)
        if patterns is not None:
            return self._scan_host_batch_filtered(chunks, overlapping, codepoints, patterns)
        if n == 1 and len(chunks[0]) <= self.SMALL_CALL_BYTES and _capi.current_kernel() in (0, 5) and self.ENGINE != "table":
            m = self._small_call(chunks[0], overlapping, codepoints)
            if m is not None:
                return m, np.array([0, m.shape[0]], dtype=np.int64)
        lens = np.fromiter((len(c) for c in chunks), dtype=np.int64, count=n)
        offs = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        total_bytes = int(offs[-1])
        with self._host_lock:
            host = self._pinned(total_bytes)
            hv = host.numpy()
            if n == 1:
                hv[:total_bytes] = np.frombuffer(chunks[0], dtype=np.uint8)
            elif total_bytes:
                hv[:total_bytes] = np.frombuffer(b"".join(chunks), dtype=np.uint8)  # one C-speed concatenation, one copy into pinned memory
            return self.scan_host(host[:total_bytes], offs, overlapping, codepoints)


    def _scan_host_batch_filtered(self, chunks: Sequence[bytes], overlapping: bool, codepoints: bool, patterns):
        """scan_host_batch with one pattern set per haystack: the haystacks are gathered into the pinned staging buffer
        with their offsets, go to the device in one copy and are scanned by scan_device with the sets (the sieve)."""
        _require_cuda()
        n = len(chunks)
        if n == 0:
            if len(list(patterns)) != 0:
                raise ValueError("patterns= needs one set of pattern ids per haystack: 0 haystacks")
            return np.zeros((0, 4), dtype=np.uint32), np.zeros(1, dtype=np.int64)
        with self._host_staged(chunks) as (data, offsets, _, _):
            flt = _host_sets(self, patterns, n, data.device)
            m, mo, _ = self.scan_device(data, offsets, overlapping, codepoints, flt=flt)
            m = m.cpu().numpy()
            return (m.view(np.uint32) if m.dtype == np.int32 else m), mo.cpu().numpy().astype(np.int64)


class StreamBatch:
    """A batch of streams on one device: data that arrives in chunks, searched across the chunk boundaries.  Stream i is
    the concatenation of the chunks fed to slot i; positions are absolute within it (int64), byte offsets, or code
    point indexes for the str class.  The rows a stream releases over all its feeds, in order, are exactly
    find_matches_as_indexes(concatenation, overlapping).  After a feed that brings a stream to F bytes, the rows
    released are those of that result with end <= F (Standard), or start + max_pattern_len <= F (the leftmost kinds:
    no later match can start before them).  The carry of every stream lives on the device (acb_stream_seams /
    acb_stream_resolve in include/acb200.h); a feed runs the sieve on the chunks as they are, never copying them."""

    _serial = __import__("itertools").count()

    def __init__(self, ac: "_Automaton", n_streams: int, overlapping: bool, codepoints: bool):
        if isinstance(n_streams, bool) or not isinstance(n_streams, int):
            raise TypeError("n_streams must be an int")
        if n_streams < 0 or n_streams > 0xFFFF_FFFE:
            raise ValueError("n_streams out of range (0 .. 2^32 - 2)")
        ac.check_overlapping(overlapping)
        halo = max(ac.max_pattern_len - 1, 0)
        if 2 * n_streams * halo > ac.WINDOW_BYTES:
            # the seams (tail || head, up to 2 * (max_pattern_len - 1) bytes per stream) are scanned in one call
            raise ValueError(f"{n_streams} streams x 2 x (max_pattern_len - 1) = {2 * n_streams * halo} seam bytes: one feed's seams "
                             f"must fit {ac.WINDOW_BYTES} bytes (WINDOW_BYTES); use fewer streams per batch")
        self._ac = ac
        self.n_streams = n_streams
        self.overlapping = bool(overlapping)
        self._codepoints = codepoints
        self.device = None     # the device of the first feed: the carry is allocated there
        self._halo = max(ac.max_pattern_len - 1, 0)
        # two workspaces of the automaton that only this batch scans with: the lists they hold are read by the resolve
        k = next(StreamBatch._serial)
        self._slots = (("stream", k, 0), ("stream", k, 1))
        self._lock = threading.Lock()
        self.last_stats = {}

    def _allocate(self, dev):
        torch = _torch()
        n = self.n_streams
        self.device = dev
        self._carry = torch.zeros((n, 4), dtype=torch.int64, device=dev)   # acb_stream_resolve's carry words
        self._tail = torch.zeros(max(n * self._halo, 1), dtype=torch.uint8, device=dev)
        self._seam = torch.empty(max(2 * n * self._halo, 1), dtype=torch.uint8, device=dev)
        self._seam_offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)

    def __del__(self):
        ac, slots = getattr(self, "_ac", None), getattr(self, "_slots", ())
        if ac is not None:
            for key in [key for key in list(ac._ws) if key[1] in slots]:
                ac._ws.pop(key, None)

    def feed_device(self, data, offsets, last=None):
        """One chunk per stream: chunk i = data[offsets[i]:offsets[i + 1]] (uint8 CUDA tensor, int64 CUDA tensor
        (n_streams + 1); an empty chunk is allowed).  `last`: None, or a bool CUDA tensor (n_streams,) -- those streams
        end with this feed, release everything and start again at position 0.  Returns (rows int64 (k, 4) = (stream,
        pattern, start, end), row_offsets int64 (n_streams + 1)), the rows of stream i at row_offsets[i]:row_offsets[i+1]."""
        torch = _torch()
        ac, n = self._ac, self.n_streams
        if not torch.is_tensor(data) or data.dtype != torch.uint8 or data.dim() != 1 or data.device.type != "cuda":
            raise TypeError("data must be a 1-D uint8 CUDA tensor")
        dev = self.device or data.device
        if data.device != dev:
            raise TypeError(f"data must be on {dev}, where this batch's streams live")
        if not torch.is_tensor(offsets) or offsets.dtype != torch.int64 or offsets.shape != (n + 1,) or offsets.device != dev:
            raise TypeError(f"offsets must be an int64 tensor of shape ({n + 1},) on {dev}")
        if last is not None and (not torch.is_tensor(last) or last.dtype != torch.bool or last.shape != (n,) or last.device != dev):
            raise TypeError(f"last must be None or a bool tensor of shape ({n},) on {dev}")
        if data.numel() > ac.WINDOW_BYTES:
            raise ValueError(f"one feed addresses at most {ac.WINDOW_BYTES} bytes (WINDOW_BYTES): feed larger data in more chunks")
        _require_cuda()
        data, offsets = data.contiguous(), offsets.contiguous()
        last_u8 = last.contiguous().view(torch.uint8) if last is not None else None
        L = ac._L
        with self._lock, torch.cuda.device(dev):
            if self.device is None:
                self._allocate(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _check(L.acb_stream_seams(ac._h, data.data_ptr(), offsets.data_ptr(), n, data.numel(), self._carry.data_ptr(),
                                      self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(), stream))
            # the overlapping lists, in bytes, of the chunks as they are and of the seams
            m_c, mo_c, tot_c = ac.scan_device(data, offsets, 2, False, ws_slot=self._slots[0])
            geometry = {k: ac.last_stats.get(k) for k in ("window", "last_level", "probes", "bloom_bytes", "ring", "task_bytes")}
            m_s, mo_s, tot_s = ac.scan_device(self._seam, self._seam_offsets, 2, False, ws_slot=self._slots[1])
            if m_c.dtype != torch.int32 or m_s.dtype != torch.int32:   # (both buffers are below WINDOW_BYTES: one call each)
                raise RuntimeError("stream search: a list came back in the windowed int64 form acb_stream_resolve cannot read")
            cap = int(tot_c) + int(tot_s)

            def ptr(t):   # an empty list is still a view of its workspace's buffer: pass that buffer's (non-null) address
                return t.data_ptr() if t.numel() else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()

            # the staging area of the selected rows (4 words per record) is not used by an overlapping search
            scratch = torch.empty(2 + 6 * n + (0 if self.overlapping else 4 * cap), dtype=torch.int64, device=dev)
            rows = torch.empty((max(cap, 1), 4), dtype=torch.int64, device=dev)
            row_offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
            rc = L.acb_stream_resolve(ac._h, ac.image(dev).data_ptr() if self._codepoints else None, data.data_ptr(), offsets.data_ptr(), n,
                                      data.numel(), last_u8.data_ptr() if last_u8 is not None else None, int(self.overlapping),
                                      int(self._codepoints), self._carry.data_ptr(), self._tail.data_ptr(), self._seam.data_ptr(),
                                      self._seam_offsets.data_ptr(), ptr(m_s), mo_s.data_ptr(), ptr(m_c), mo_c.data_ptr(),
                                      scratch.data_ptr(), rows.data_ptr(), row_offsets.data_ptr(), stream)
            if rc != _capi.ACB_OK:
                raise (ValueError if rc == _capi.ACB_EUNSUPPORTED else RuntimeError)(_capi.last_error())
            k = int(row_offsets[n].item())
            records, held = scratch[:2].tolist()
        self.last_stats = {"engine": "sieve", "mode": "stream", **geometry, "seam_bytes": int(self._seam_offsets[n].item()),
                           "records": records, "released": k, "held": held}
        ac.last_stats = dict(self.last_stats)
        return rows[:k], row_offsets


class Stream:
    """One stream fed from the host: a StreamBatch of one, with its own pinned staging buffer for the chunks (so a feed
    does not wait for the automaton's other host-staged calls, nor they for it)."""

    def __init__(self, ac: "_Automaton", overlapping: bool, codepoints: bool):
        self._batch = StreamBatch(ac, 1, overlapping, codepoints)
        self._ac = ac
        self._codepoints = codepoints
        self._offs = None
        self._pinned = None
        self._lock = threading.Lock()
        self._done = False

    @property
    def last_stats(self):
        return self._batch.last_stats

    def feed(self, chunk):
        """The next chunk (a str for AhoCorasick, a bytes-like object for BytesAhoCorasick) -> the rows
        [(pattern, start, end), ...] this feed releases."""
        if self._codepoints:
            if not isinstance(chunk, str):
                raise TypeError("argument 'chunk': 'str' expected")
            return self._feed(chunk.encode("utf-8"), False)
        return self._feed(_as_buffer_bytes(chunk), False)

    def _feed(self, chunk, last: bool):
        torch = _torch()
        if self._done:
            raise RuntimeError("the stream is finished: feed after finish()")
        n = len(chunk)
        if n > self._ac.WINDOW_BYTES:
            raise ValueError(f"one feed addresses at most {self._ac.WINDOW_BYTES} bytes (WINDOW_BYTES): feed larger data in more chunks")
        torch = _require_cuda()
        dev = self._batch.device or torch.device("cuda", torch.cuda.current_device())
        if self._offs is None:
            self._offs = torch.zeros(2, dtype=torch.int64, device=dev)
        with self._lock:   # the staging buffer is reused once the feed has synchronised (feed_device reads its row count)
            if self._pinned is None or self._pinned.numel() < n:
                self._pinned = torch.empty(max(n, 1 << 16), dtype=torch.uint8, pin_memory=True)
            host = self._pinned
            if n:
                host.numpy()[:n] = np.frombuffer(chunk, dtype=np.uint8)
            d = host[:n].to(dev, non_blocking=True)
            self._offs[1] = n
            rows, _ = self._batch.feed_device(d, self._offs, torch.ones(1, dtype=torch.bool, device=dev) if last else None)
            rows = rows.cpu().numpy()
        if last:
            self._done = True
        return list(zip(rows[:, 1].tolist(), rows[:, 2].tolist(), rows[:, 3].tolist()))

    def finish(self):
        """The rows still held; ends the stream."""
        return self._feed(b"", True)


class _QueryStreamBatch(StreamBatch):
    """The stream forms of is_match, find_first and count_matches: one answer per stream after every feed, without the
    rows.  They share StreamBatch's slots, limits, carry and seams (acb_stream_seams, then the kind's scans and resolve,
    then acb_stream_advance; see include/acb200.h).  A feed with `last` returns those streams' final answers and
    starts their slots again."""

    MODE = ""
    POSITIONS = False   # answers with positions (code points are carried for the str class)
    _flt = None         # each stream's pattern set (is_match and find_first): (PatternSets, set index (n_streams,))

    def _feed_args(self, data, offsets, last):
        torch = _torch()
        n = self.n_streams
        if not torch.is_tensor(data) or data.dtype != torch.uint8 or data.dim() != 1 or data.device.type != "cuda":
            raise TypeError("data must be a 1-D uint8 CUDA tensor")
        dev = self.device or data.device
        if data.device != dev:
            raise TypeError(f"data must be on {dev}, where this batch's streams live")
        if not torch.is_tensor(offsets) or offsets.dtype != torch.int64 or offsets.shape != (n + 1,) or offsets.device != dev:
            raise TypeError(f"offsets must be an int64 tensor of shape ({n + 1},) on {dev}")
        if last is not None and (not torch.is_tensor(last) or last.dtype != torch.bool or last.shape != (n,) or last.device != dev):
            raise TypeError(f"last must be None or a bool tensor of shape ({n},) on {dev}")
        if data.numel() > self._ac.WINDOW_BYTES:
            raise ValueError(f"one feed addresses at most {self._ac.WINDOW_BYTES} bytes (WINDOW_BYTES): feed larger data in more chunks")
        if self._flt is not None and dev != self._flt[0].device:
            raise TypeError(f"data must be on {self._flt[0].device}, where this batch's pattern sets live")
        _require_cuda()
        return dev, data.contiguous(), offsets.contiguous(), (last.contiguous().view(torch.uint8) if last is not None else None)

    def feed_device(self, data, offsets, last=None):
        """One chunk per stream, as StreamBatch.feed_device takes them -> the answers after this feed (a CUDA tensor,
        see the subclass)."""
        torch = _torch()
        dev, data, offsets, last_u8 = self._feed_args(data, offsets, last)
        ac, L = self._ac, self._ac._L
        with self._lock, ac._lock, torch.cuda.device(dev):
            if self.device is None:
                self._allocate(dev)
                self._allocate_query(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _check(L.acb_stream_seams(ac._h, data.data_ptr(), offsets.data_ptr(), self.n_streams, data.numel(), self._carry.data_ptr(),
                                      self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(), stream))
            out, stats = self._query(dev, data, offsets, last_u8, stream)
            cp = self._codepoints and self.POSITIONS
            scratch = torch.empty(6 * self.n_streams if cp else 1, dtype=torch.int64, device=dev)
            _check(L.acb_stream_advance(ac._h, data.data_ptr(), offsets.data_ptr(), self.n_streams, data.numel(),
                                        last_u8.data_ptr() if last_u8 is not None else None, int(cp), self._carry.data_ptr(),
                                        self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(), scratch.data_ptr(), stream))
            task_bytes = int(ac._plan(data, max(self.n_streams, 1)).task_bytes)
            self.last_stats = {"engine": "sieve", "mode": self.MODE, **ac.sieve_geometry(dev, task_bytes),
                               "seam_bytes": int(self._seam_offsets[self.n_streams].item()), **stats, **ac._set_stats(self._flt)}
        ac.last_stats = dict(self.last_stats)
        return out

    def _skips(self, scratch):
        """tasks_skipped / windows_skipped of an acb_any_match or acb_find_first scratch (one synchronisation)."""
        _, skipped, windows = scratch.tolist()
        return {"tasks_skipped": skipped, "windows_skipped": windows}


class IsMatchStreamBatch(_QueryStreamBatch):
    """is_match per stream: feed_device returns a bool CUDA tensor (n_streams,), flag i = is_match(the stream's
    concatenation so far).  A flag stays set until its stream ends; the chunks of a flagged stream are skipped by the
    scan's task skip, so a stream that has matched costs almost nothing to keep feeding."""

    MODE = "is_match_stream"

    def _allocate_query(self, dev):
        self._flags = _torch().zeros(self.n_streams, dtype=_torch().bool, device=dev)

    def _query(self, dev, data, offsets, last_u8, stream):
        torch = _torch()
        ac, L, n = self._ac, self._ac._L, self.n_streams
        sieve_t, _ = ac.sieve(dev)
        scratch = torch.empty((2, 3), dtype=torch.int64, device=dev)
        # the seams first: a stream whose match crosses the cut then has its chunk skipped
        for k, (b, o) in enumerate(((self._seam, self._seam_offsets), (data, offsets))):
            _check(L.acb_any_match_filtered(ac._h, sieve_t.data_ptr(), b.data_ptr(), o.data_ptr(), n, b.numel(), self._flags.data_ptr(),
                                            scratch[k].data_ptr(), _filter_struct(self._flt), stream))
        out = self._flags.clone()
        if last_u8 is not None:
            self._flags.masked_fill_(last_u8.view(torch.bool), False)
        return out, {**self._skips(scratch[1]), "flagged": int(out.sum().item())}


class FindFirstStreamBatch(_QueryStreamBatch):
    """find_first per stream: feed_device returns an int64 CUDA tensor (n_streams, 3): row i is find_first of the
    stream's whole concatenation, (pattern, start, end), as soon as no later data can change it -- Standard at once,
    the leftmost kinds once start + max_pattern_len <= the bytes fed, every stream on `last` -- and (-1, -1, -1) before
    that (or after `last` when the stream had no match).  Byte offsets, or code point indexes for the str class."""

    MODE = "find_first_stream"
    POSITIONS = True

    def _allocate_query(self, dev):
        torch = _torch()
        n = self.n_streams
        self._best = torch.zeros((n, 6), dtype=torch.int64, device=dev)
        self._keys = torch.full((2, n), -1, dtype=torch.int64, device=dev)   # seam keys, chunk keys: ~0 = scan

    def _query(self, dev, data, offsets, last_u8, stream):
        torch = _torch()
        ac, L, n = self._ac, self._ac._L, self.n_streams
        ac.first_keys(self._seam, self._seam_offsets, self._keys[0], self._flt)
        chunk_scratch = ac.first_keys(data, offsets, self._keys[1], self._flt)
        scratch = torch.empty(2 + 12 * n, dtype=torch.int64, device=dev)
        rows = torch.empty((n, 3), dtype=torch.int64, device=dev)
        _check(L.acb_stream_first_resolve_filtered(ac._h, ac.sieve(dev)[0].data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                                                   last_u8.data_ptr() if last_u8 is not None else None, int(self._codepoints),
                                                   self._carry.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(),
                                                   self._seam.numel(), self._keys[0].data_ptr(), self._keys[1].data_ptr(), self._best.data_ptr(),
                                                   scratch.data_ptr(), rows.data_ptr(), _filter_struct(self._flt), stream))
        return rows, {**self._skips(chunk_scratch), "pending": int(scratch[1].item())}


class CountStreamBatch(_QueryStreamBatch):
    """count_matches per stream: feed_device returns an int64 CUDA tensor (n_streams,), count i = the number of rows the
    stream search (stream_batch, same `overlapping`) would have released so far; after `last`, count_matches of the
    stream's concatenation.  Overlapping: the sieve's count mode on the chunks plus the seam records that cross the
    cut, no rows.  Non-overlapping: the stream search's two lists, with the selection counted (one thread per stream, or
    the whole grid for a stream with more than ACB_LONG_STRETCH records)."""

    MODE = "count_stream"

    def _allocate_query(self, dev):
        self._running = _torch().zeros(self.n_streams, dtype=_torch().int64, device=dev)

    def _query(self, dev, data, offsets, last_u8, stream):
        torch = _torch()
        ac, L, n = self._ac, self._ac._L, self.n_streams
        m_s, mo_s, tot_s = ac.scan_device(self._seam, self._seam_offsets, 2, False, ws_slot=self._slots[1])
        if self.overlapping:
            chunk_counts = torch.zeros(n, dtype=torch.int64, device=dev)
            scratch = torch.empty(3, dtype=torch.int64, device=dev)
            _check(L.acb_count_overlapping(ac._h, ac.sieve(dev)[0].data_ptr(), data.data_ptr(), offsets.data_ptr(), n, data.numel(),
                                           chunk_counts.data_ptr(), scratch.data_ptr(), stream))
            m_c = mo_c = None
            words = 4
        else:
            m_c, mo_c, tot_c = ac.scan_device(data, offsets, 2, False, ws_slot=self._slots[0])
            chunk_counts = None
            words = 4 + 6 * n + 4 * (int(tot_c) + int(tot_s))
        if m_s.dtype != torch.int32 or (m_c is not None and m_c.dtype != torch.int32):
            raise RuntimeError("stream count: a list came back in the windowed int64 form acb_stream_count cannot read")

        def ptr(t):   # an empty list is still a view of its workspace's buffer: pass that buffer's (non-null) address
            return t.data_ptr() if t.numel() else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()

        scratch = torch.empty(words, dtype=torch.int64, device=dev)
        counts = torch.empty(n, dtype=torch.int64, device=dev)
        rc = L.acb_stream_count(ac._h, data.data_ptr(), offsets.data_ptr(), n, data.numel(), last_u8.data_ptr() if last_u8 is not None else None,
                                int(self.overlapping), self._carry.data_ptr(), self._seam_offsets.data_ptr(), ptr(m_s), mo_s.data_ptr(),
                                ptr(m_c) if m_c is not None else None, mo_c.data_ptr() if mo_c is not None else None,
                                chunk_counts.data_ptr() if chunk_counts is not None else None, self._running.data_ptr(), counts.data_ptr(),
                                scratch.data_ptr(), words, stream)
        if rc != _capi.ACB_OK:
            raise (ValueError if rc == _capi.ACB_EUNSUPPORTED else RuntimeError)(_capi.last_error())
        records, held, long_stretches = scratch[:3].tolist()
        return counts, {"records": records, "held": held, "long_stretches": long_stretches}


class MaskStreamBatch(_QueryStreamBatch):
    """Match masks per stream: after each feed, the flags of the positions no later data can change.  With halo =
    max_pattern_len - 1 and F the bytes stream i has been fed, it has released the positions whose first byte lies below
    R = max(0, F - halo) (all of them on `last`, after which the slot starts again at 0).  A released flag is final: it
    equals match_mask_device of the whole concatenation at that position (overlapping or not; with pattern sets, the
    stream's set).  feed_device returns (flags bool (k,), flag_offsets int64 (n_streams + 1), flag_starts int64
    (n_streams,)): stream i's flags are flags[flag_offsets[i]:flag_offsets[i + 1]], for its positions flag_starts[i],
    flag_starts[i] + 1, ...  A flag per byte, or per token id (stride = ACB_TOKEN_BYTES) for TokenAhoCorasick.

    Overlapping: the sieve's cover mode on the chunks and on the seams, no list.  Non-overlapping: the stream search's
    two list scans and resolve, then acb_stream_mask_rows.  Then acb_stream_mask_emit (include/acb200.h)."""

    MODE = "match_mask_stream"

    def __init__(self, ac: "_Automaton", n_streams: int, overlapping: bool, stride: int = 1):
        super().__init__(ac, n_streams, overlapping, codepoints=False)
        self._stride = stride

    def _allocate_query(self, dev):
        torch = _torch()
        size = max(self.n_streams * self._halo, 1)
        self._held = (torch.zeros(size, dtype=torch.uint8, device=dev), torch.zeros(size, dtype=torch.uint8, device=dev))

    def feed_device(self, data, offsets, last=None):
        torch = _torch()
        dev, data, offsets, last_u8 = self._feed_args(data, offsets, last)
        ac, L, n = self._ac, self._ac._L, self.n_streams
        flt = _filter_struct(self._flt)
        with self._lock, ac._lock, torch.cuda.device(dev):
            if self.device is None:
                self._allocate(dev)
                self._allocate_query(dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            last_p = last_u8.data_ptr() if last_u8 is not None else None
            _check(L.acb_stream_seams(ac._h, data.data_ptr(), offsets.data_ptr(), n, data.numel(), self._carry.data_ptr(),
                                      self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(), stream))
            chunk_bits = torch.zeros(max((data.numel() + 31) // 32, 1), dtype=torch.int32, device=dev)
            seam_bits = torch.zeros(max((self._seam.numel() + 31) // 32, 1), dtype=torch.int32, device=dev)
            if self.overlapping:
                carry_before = self._carry   # the emit runs before the advance
                sieve_t = ac.sieve(dev)[0]
                scratch = torch.empty(3, dtype=torch.int64, device=dev)
                for b, o, w in ((data, offsets, chunk_bits), (self._seam, self._seam_offsets, seam_bits)):
                    _check(L.acb_match_mask_overlapping_filtered(ac._h, sieve_t.data_ptr(), b.data_ptr(), o.data_ptr(), n, b.numel(),
                                                                 w.data_ptr(), 0, scratch.data_ptr(), flt, stream))
                stats = {}
            else:
                # the overlapping lists, in bytes, of the chunks as they are and of the seams (as StreamBatch.feed_device)
                m_c, mo_c, tot_c = ac.scan_device(data, offsets, 2, False, ws_slot=self._slots[0], flt=self._flt)
                m_s, mo_s, tot_s = ac.scan_device(self._seam, self._seam_offsets, 2, False, ws_slot=self._slots[1], flt=self._flt)
                if m_c.dtype != torch.int32 or m_s.dtype != torch.int32:
                    raise RuntimeError("match-mask stream: a list came back in the windowed int64 form acb_stream_resolve cannot read")
                cap = int(tot_c) + int(tot_s)

                def ptr(t):   # an empty list is still a view of its workspace's buffer: pass that buffer's (non-null) address
                    return t.data_ptr() if t.numel() else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()

                carry_before = self._carry.clone()   # the resolve moves the carry (and zeroes it on `last`)
                scratch = torch.empty(2 + 6 * n + 4 * cap, dtype=torch.int64, device=dev)
                rows = torch.empty((max(cap, 1), 4), dtype=torch.int64, device=dev)
                row_offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
                _check(L.acb_stream_resolve(ac._h, None, data.data_ptr(), offsets.data_ptr(), n, data.numel(), last_p, 0, 0,
                                            self._carry.data_ptr(), self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(),
                                            ptr(m_s), mo_s.data_ptr(), ptr(m_c), mo_c.data_ptr(), scratch.data_ptr(), rows.data_ptr(),
                                            row_offsets.data_ptr(), stream))
                _check(L.acb_stream_mask_rows(offsets.data_ptr(), n, carry_before.data_ptr(), self._seam_offsets.data_ptr(), rows.data_ptr(),
                                              row_offsets.data_ptr(), chunk_bits.data_ptr(), seam_bits.data_ptr(), stream))
                stats = {"records": scratch[0]}
            flags = torch.empty(max(data.numel() + n * self._halo, 1), dtype=torch.bool, device=dev)
            flag_offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
            flag_starts = torch.empty(n, dtype=torch.int64, device=dev)
            held_in, held_out = self._held
            rc = L.acb_stream_mask_emit(ac._h, offsets.data_ptr(), n, last_p, int(self.overlapping), self._stride, carry_before.data_ptr(),
                                        self._seam_offsets.data_ptr(), chunk_bits.data_ptr(), seam_bits.data_ptr(), held_in.data_ptr(),
                                        held_out.data_ptr(), flags.data_ptr(), flag_offsets.data_ptr(), flag_starts.data_ptr(), stream)
            if rc != _capi.ACB_OK:
                raise (ValueError if rc == _capi.ACB_EUNSUPPORTED else RuntimeError)(_capi.last_error())
            self._held = (held_out, held_in)
            if self.overlapping:
                _check(L.acb_stream_advance(ac._h, data.data_ptr(), offsets.data_ptr(), n, data.numel(), last_p, 0, self._carry.data_ptr(),
                                            self._tail.data_ptr(), self._seam.data_ptr(), self._seam_offsets.data_ptr(), None, stream))
            counts = torch.stack([flag_offsets[n], self._seam_offsets[n], self._carry[:, 2].sum(), *stats.values()]).tolist()
            k, seam_bytes, held = counts[:3]
            task_bytes = int(ac._plan(data, max(n, 1)).task_bytes)
            self.last_stats = {"engine": "sieve", "mode": self.MODE, **ac.sieve_geometry(dev, task_bytes), "seam_bytes": seam_bytes,
                               "released": k, "held": held, **dict(zip(stats, counts[3:])), **ac._set_stats(self._flt)}
        ac.last_stats = dict(self.last_stats)
        return flags[:k], flag_offsets, flag_starts


class QueryStream:
    """One query stream fed from the host (a query batch of one, with its own pinned staging buffer): feed(chunk) and
    finish() return the answer after the feed (see the batch classes); finish() ends the stream."""

    def __init__(self, batch: _QueryStreamBatch, answer):
        self._batch = batch
        self._answer = answer
        self._codepoints = batch._codepoints
        self._offs = None
        self._pinned = None
        self._lock = threading.Lock()
        self._done = False

    @property
    def last_stats(self):
        return self._batch.last_stats

    def feed(self, chunk):
        """The next chunk (a str for AhoCorasick, a bytes-like object for BytesAhoCorasick) -> the answer so far."""
        if self._codepoints:
            if not isinstance(chunk, str):
                raise TypeError("argument 'chunk': 'str' expected")
            return self._feed(chunk.encode("utf-8"), False)
        return self._feed(_as_buffer_bytes(chunk), False)

    def finish(self):
        """The final answer; ends the stream."""
        return self._feed(b"", True)

    def _feed(self, chunk, last: bool):
        if self._done:
            raise RuntimeError("the stream is finished: feed after finish()")
        n = len(chunk)
        ac = self._batch._ac
        if n > ac.WINDOW_BYTES:
            raise ValueError(f"one feed addresses at most {ac.WINDOW_BYTES} bytes (WINDOW_BYTES): feed larger data in more chunks")
        torch = _require_cuda()
        dev = self._batch.device or torch.device("cuda", torch.cuda.current_device())
        if self._offs is None:
            self._offs = torch.zeros(2, dtype=torch.int64, device=dev)
        with self._lock:   # the staging buffer is reused once the answer is on the host
            if self._pinned is None or self._pinned.numel() < n:
                self._pinned = torch.empty(max(n, 1 << 16), dtype=torch.uint8, pin_memory=True)
            host = self._pinned
            if n:
                host.numpy()[:n] = np.frombuffer(chunk, dtype=np.uint8)
            d = host[:n].to(dev, non_blocking=True)
            self._offs[1] = n
            out = self._batch.feed_device(d, self._offs, torch.ones(1, dtype=torch.bool, device=dev) if last else None)
            ans = self._answer(out[0].tolist())
        if last:
            self._done = True
        return ans


class MaskStream(QueryStream):
    """One match-mask stream fed from the host (a MaskStreamBatch of one): feed(chunk) returns the runs [(start, end),
    ...] of covered positions inside the range this feed released, clipped to it, in the class's unit (code points,
    bytes or tokens); finish() returns the rest and ends the stream.  Merging every feed's runs that touch at a feed
    boundary gives match_spans(concatenation, overlapping, patterns).  For str chunks a code point is released with its
    lead byte: the stream keeps the bytes fed but not released, to tell lead bytes from continuation bytes."""

    def __init__(self, batch: MaskStreamBatch, codepoints: bool):
        super().__init__(batch, None)
        self._codepoints = codepoints
        self._pending = np.zeros(0, dtype=np.uint8)   # str: the bytes [R, F), fed but not released
        self._released = 0

    @property
    def released(self) -> int:
        """The positions released so far (code points, bytes or tokens)."""
        return self._released

    def _feed(self, chunk, last: bool):
        if self._done:
            raise RuntimeError("the stream is finished: feed after finish()")
        n = len(chunk)
        ac = self._batch._ac
        if n > ac.WINDOW_BYTES:
            raise ValueError(f"one feed addresses at most {ac.WINDOW_BYTES} bytes (WINDOW_BYTES): feed larger data in more chunks")
        torch = _require_cuda()
        dev = self._batch.device or torch.device("cuda", torch.cuda.current_device())
        if self._offs is None:
            self._offs = torch.zeros(2, dtype=torch.int64, device=dev)
        with self._lock:   # the staging buffer is reused once the flags are on the host
            if self._pinned is None or self._pinned.numel() < n:
                self._pinned = torch.empty(max(n, 1 << 16), dtype=torch.uint8, pin_memory=True)
            host = self._pinned
            if n:
                host.numpy()[:n] = np.frombuffer(chunk, dtype=np.uint8)
            d = host[:n].to(dev, non_blocking=True)
            self._offs[1] = n
            flags, _, _ = self._batch.feed_device(d, self._offs, torch.ones(1, dtype=torch.bool, device=dev) if last else None)
            flags = flags.cpu().numpy()
            if self._codepoints:   # a flag per byte: keep those of lead bytes, one per code point
                text = np.concatenate([self._pending, host.numpy()[:n]])
                self._pending = text[flags.size:]
                flags = flags[(text[:flags.size] & 0xC0) != 0x80]
        start = self._released   # each feed's positions follow the last feed's
        self._released += flags.size
        if last:
            self._done = True
        prev = np.concatenate([[False], flags])
        nxt = np.concatenate([flags, [False]])
        return list(zip((np.flatnonzero(nxt & ~prev) + start).tolist(), (np.flatnonzero(prev & ~nxt) + start).tolist()))


def _mask_stream_batch(ac, n_streams: int, overlapping: bool, pattern_sets=None, set_index=None, stride: int = 1) -> MaskStreamBatch:
    """A match-mask batch; pattern_sets= / set_index= fix each stream's pattern set for the batch's life."""
    batch = MaskStreamBatch(ac, n_streams, overlapping, stride)
    if pattern_sets is not None or set_index is not None:
        dev = pattern_sets.device if isinstance(pattern_sets, PatternSets) else None
        batch._flt = _filter_args(ac, pattern_sets, set_index, n_streams, dev)
    return batch


def _mask_stream(ac, overlapping: bool, codepoints: bool, patterns=None, stride: int = 1) -> MaskStream:
    """A host-fed match-mask stream; `patterns`: the stream's pattern ids, or None."""
    if patterns is None:
        return MaskStream(_mask_stream_batch(ac, 1, overlapping, stride=stride), codepoints)
    torch = _require_cuda()
    ps = PatternSets(ac, [patterns])
    return MaskStream(_mask_stream_batch(ac, 1, overlapping, ps, torch.zeros(1, dtype=torch.int32, device=ps.device), stride), codepoints)


def _first_answer(row):
    return tuple(row) if row[0] >= 0 else None


def _query_stream_batch(ac, kind: str, n_streams: int, overlapping: bool, codepoints: bool, pattern_sets=None,
                        set_index=None) -> _QueryStreamBatch:
    """A query batch; is_match and find_first take each stream's pattern set (fixed for the batch's life)."""
    cls = {"is_match": IsMatchStreamBatch, "find_first": FindFirstStreamBatch, "count": CountStreamBatch}[kind]
    batch = cls(ac, n_streams, overlapping, codepoints)
    if pattern_sets is not None or set_index is not None:
        dev = pattern_sets.device if isinstance(pattern_sets, PatternSets) else None
        batch._flt = _filter_args(ac, pattern_sets, set_index, n_streams, dev)
    return batch


def _query_stream(ac, kind: str, overlapping: bool, codepoints: bool, patterns=None) -> QueryStream:
    """A host-fed query stream; `patterns`: the stream's pattern ids (is_match and find_first), or None."""
    answer = {"is_match": bool, "find_first": _first_answer, "count": int}[kind]
    if patterns is None:
        return QueryStream(_query_stream_batch(ac, kind, 1, overlapping, codepoints), answer)
    torch = _require_cuda()
    ps = PatternSets(ac, [patterns])
    return QueryStream(_query_stream_batch(ac, kind, 1, overlapping, codepoints, ps, torch.zeros(1, dtype=torch.int32, device=ps.device)),
                       answer)


def _as_buffer_bytes(obj) -> bytes:
    """reference PyBufferBytes::try_from (src/lib.rs:281-302): 1-D, C-contiguous u8 buffer."""
    if isinstance(obj, str):
        raise TypeError("a bytes-like object is required, not 'str'")
    try:
        mv = memoryview(obj)
    except TypeError as e:
        raise TypeError(str(e)) from None
    if mv.ndim > 1:
        raise TypeError("Only one-dimensional sequences are supported")
    if not mv.c_contiguous:
        raise TypeError("Must be a contiguous sequence of bytes")
    if mv.itemsize != 1 or mv.format not in ("B", "b", "c"):
        raise BufferError("buffer contents are not compatible with u8")
    # zero-copy like the reference's PyBufferBytes (src/lib.rs:304-340): the caller's memory is read in place (one copy,
    # into the pinned staging buffer the H2D transfer starts from); as there, the caller must not mutate it meanwhile
    return obj if isinstance(obj, bytes) else (mv if mv.format == "B" else mv.cast("B"))


def _tuples(m: np.ndarray):
    return list(zip(m[:, 1].tolist(), m[:, 2].tolist(), m[:, 3].tolist()))


def spans_from_words(words: np.ndarray, offs: np.ndarray, text: Optional[np.ndarray] = None, unit: int = 1):
    """A packed mask (u32 words, bit p % 32 of word p // 32 = byte p; any 4-byte integer dtype) over the haystacks
    [offs[h], offs[h + 1]) -> one list of (start, end) per haystack: its maximal runs of covered bytes, cut at haystack
    boundaries, haystack-relative.  With `text` (the batch's UTF-8 bytes) positions are code points: a byte position
    maps to the number of lead bytes before it.  Else they are bytes divided by `unit` (3 for token ids)."""
    offs = np.asarray(offs, dtype=np.int64)
    n, total = len(offs) - 1, int(offs[-1])
    bits = np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")[:total].astype(bool)
    bits[:int(offs[0])] = False
    # a run starts where a covered byte follows an uncovered one or a haystack start; it ends symmetrically
    cut = np.zeros(total + 1, dtype=bool)
    cut[offs] = True
    prev = np.concatenate([[False], bits])
    nxt = np.concatenate([bits, [False]])
    starts = np.flatnonzero(nxt & (~prev | cut))
    ends = np.flatnonzero(prev & (~nxt | cut))
    hay = np.searchsorted(offs, starts, side="right") - 1
    if text is not None:
        lead = np.zeros(total + 1, dtype=np.int64)
        np.cumsum((np.asarray(text[:total]) & 0xC0) != 0x80, out=lead[1:])
        base = lead[offs[hay]]
        s, e = lead[starts] - base, lead[ends] - base
    else:
        base = offs[hay]
        s, e = (starts - base) // unit, (ends - base) // unit
    bounds = np.searchsorted(hay, np.arange(n + 1), side="left")
    pairs = list(zip(s.tolist(), e.tolist()))
    return [pairs[bounds[h]:bounds[h + 1]] for h in range(n)]


def _one_set(patterns):
    """A single-haystack host call's patterns= -> the per-haystack list the host batches take (None stays None)."""
    return None if patterns is None else [patterns]


def _batch_sets(patterns, n: int):
    """A host batch's patterns= (one iterable of ids per haystack) -> a list of n of them (None stays None)."""
    if patterns is None:
        return None
    sets = list(patterns)
    if len(sets) != n:
        raise ValueError(f"patterns= needs one set of pattern ids per haystack: {n} haystacks, {len(sets)} sets")
    return sets


class _PatternSetMethods:
    """pattern_sets() and the device-call check of (pattern_sets, set_index), shared by the three classes."""

    def pattern_sets(self, sets, device=None) -> PatternSets:
        """Pattern sets for the pattern_sets= / set_index= arguments: `sets` is a list of iterables of pattern ids or a
        (G, P) bool tensor; packed once into a bitset on `device` (default: the current CUDA device).  Ids outside
        [0, P), G == 0 or a tensor of another shape raise ValueError."""
        return PatternSets(self._ac, sets, device)

    def _device_filter(self, data, offsets, pattern_sets, set_index):
        return _filter_args(self._ac, pattern_sets, set_index, offsets.numel() - 1, data.device)


class AhoCorasick(_PatternSetMethods):
    """Search for multiple pattern strings against a haystack string
    (reference: src/lib.rs:15-33, 134-273).

    * ``patterns``: any iterable of non-empty ``str``.
    * ``matchkind``: ``MatchKind.Standard`` (default), ``LeftmostFirst`` or ``LeftmostLongest``.
    * ``store_patterns``: keep references to the patterns to speed up
      ``find_matches_as_strings``; ``None`` = store iff total length <= 4096 code points.
    * ``implementation``: ``Implementation`` hint or ``None``.
    """

    def __init__(self, patterns: Iterable[str], matchkind: MatchKind = MatchKind.Standard,
                 store_patterns: Optional[bool] = None, implementation: Optional[Implementation] = None):
        if not isinstance(matchkind, MatchKind):
            raise TypeError("matchkind must be a MatchKind")
        if implementation is not None and not isinstance(implementation, Implementation):
            raise TypeError("implementation must be an Implementation or None")
        it = iter(patterns)  # TypeError for non-iterables, like try_iter()? at src/lib.rs:147
        strs = []
        encoded = []
        total = 0
        decide = store_patterns is None
        store = True if decide else bool(store_patterns)
        for p in it:
            if not isinstance(p, str):
                raise TypeError(f"'{type(p).__name__}' object cannot be converted to 'PyString'")
            if p == "":
                raise ValueError("You passed in an empty string as a pattern")
            try:
                b = p.encode("utf-8")
            except UnicodeEncodeError:
                break  # reference quirk: a pattern that is not valid UTF-8 silently ends ingestion (src/lib.rs:200-203)
            if decide and store:
                total += len(p)
                if total > 4096:
                    store = False
                    strs = []
            if store:
                strs.append(p)
            encoded.append(b)
        self._patterns = strs if store else None
        self._ac = _Automaton(encoded, matchkind, implementation)

    def find_matches_as_indexes(self, haystack: str, overlapping: bool = False, patterns=None):
        """-> list of (pattern index, start, end) in code points (src/lib.rs:229-249).  `patterns`: search only for
        these pattern ids (as an automaton of those patterns would; ids stay the full automaton's)."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        m, _ = self._ac.scan_host_batch([haystack.encode("utf-8")], overlapping, codepoints=True, patterns=_one_set(patterns))
        return _tuples(m)

    def find_matches_as_strings(self, haystack: str, overlapping: bool = False, patterns=None):
        """-> list of matched patterns (src/lib.rs:253-272).  `patterns`: as for find_matches_as_indexes."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        m, _ = self._ac.scan_host_batch([haystack.encode("utf-8")], overlapping, codepoints=True, patterns=_one_set(patterns))
        if self._patterns is not None:
            pats = self._patterns
            return [pats[i] for i in m[:, 1].tolist()]
        return [haystack[s:e] for s, e in zip(m[:, 2].tolist(), m[:, 3].tolist())]

    # ---- additions: batches ------------------------------------------------------
    def find_matches_as_indexes_batch(self, haystacks: Sequence[str], overlapping: bool = False, patterns=None):
        """One list of (pattern, start, end) per haystack, each exactly what
        ``find_matches_as_indexes`` returns for it (`patterns`: one iterable of ids per haystack)."""
        self._ac.check_overlapping(overlapping)
        m, offs = self._ac.scan_host_batch([h.encode("utf-8") for h in haystacks], overlapping, codepoints=True,
                                           patterns=_batch_sets(patterns, len(haystacks)))
        t = _tuples(m)
        return [t[offs[i]:offs[i + 1]] for i in range(len(haystacks))]

    def scan_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None, **kw):
        """Device-resident UTF-8 batch -> (matches, match_offsets, total); code point indexes.  pattern_sets= /
        set_index=: haystack i searches only for the patterns of set set_index[i]."""
        self._ac.check_overlapping(overlapping)
        return self._ac.scan_device(data, offsets, overlapping, codepoints=True,
                                    flt=self._device_filter(data, offsets, pattern_sets, set_index), **kw)

    # ---- additions: yes / no per haystack (the crate's AhoCorasick::is_match) ------------------------------
    def is_match(self, haystack: str, patterns=None) -> bool:
        """Does any pattern occur in `haystack`?  The same for every match kind, so there is no `overlapping`."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        return self._ac.any_host_batch([haystack.encode("utf-8")], _one_set(patterns))[0]

    def is_match_batch(self, haystacks: Sequence[str], patterns=None) -> list:
        """``is_match`` for each haystack, in one transfer and one scan."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        return self._ac.any_host_batch([h.encode("utf-8") for h in hays], _batch_sets(patterns, len(hays)))

    def is_match_device(self, data, offsets, out=None, sync: bool = True, pattern_sets=None, set_index=None):
        """Device-resident UTF-8 batch -> bool tensor (n,) on its device (see _Automaton.any_device)."""
        return self._ac.any_device(data, offsets, out, sync, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: the first match per haystack (the crate's AhoCorasick::find) ---------------------------------
    def find_first(self, haystack: str, patterns=None):
        """-> (pattern index, start, end) in code points, or None: ``find_matches_as_indexes(haystack)[0]``, found
        without the rest of the list."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        return self._ac.first_host_batch([haystack.encode("utf-8")], codepoints=True, patterns=_one_set(patterns))[0]

    def find_first_batch(self, haystacks: Sequence[str], patterns=None) -> list:
        """``find_first`` for each haystack, in one transfer and one scan."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        return self._ac.first_host_batch([h.encode("utf-8") for h in hays], codepoints=True, patterns=_batch_sets(patterns, len(hays)))

    def find_first_device(self, data, offsets, pattern_sets=None, set_index=None):
        """Device-resident UTF-8 batch -> int64 tensor (n, 3) of (pattern, start, end) in code points, -1 rows where a
        haystack has no match (see _Automaton.first_device)."""
        return self._ac.first_device(data, offsets, codepoints=True, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: match counts per haystack ------------------------------------------------------------------
    def count_matches(self, haystack: str, overlapping: bool = False, patterns=None) -> int:
        """-> ``len(find_matches_as_indexes(haystack, overlapping))``, counted without building the list."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.count_host_batch([haystack.encode("utf-8")], overlapping, _one_set(patterns))[0]

    def count_matches_batch(self, haystacks: Sequence[str], overlapping: bool = False, patterns=None) -> list:
        """``count_matches`` for each haystack, in one transfer and one scan."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.count_host_batch([h.encode("utf-8") for h in hays], overlapping, _batch_sets(patterns, len(hays)))

    def count_matches_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident UTF-8 batch -> int64 tensor (n,) of match counts (see _Automaton.count_device)."""
        self._ac.check_overlapping(overlapping)
        return self._ac.count_device(data, offsets, overlapping, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: which positions lie inside a match ---------------------------------------------------------
    def match_spans(self, haystack: str, overlapping: bool = False, patterns=None) -> list:
        """-> [(start, end), ...] in code points: the maximal runs of code points that lie inside some match of
        ``find_matches_as_indexes(haystack, overlapping)``.  Overlapping or touching matches merge into one span."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.spans_host_batch([haystack.encode("utf-8")], overlapping, True, _one_set(patterns))[0]

    def match_spans_batch(self, haystacks: Sequence[str], overlapping: bool = False, patterns=None) -> list:
        """``match_spans`` for each haystack, in one transfer and one scan; a span never crosses a haystack boundary."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.spans_host_batch([h.encode("utf-8") for h in hays], overlapping, True, _batch_sets(patterns, len(hays)))

    def match_mask_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident UTF-8 batch -> bool tensor of data's shape: byte p is True when it lies inside a match of its
        haystack (every byte of a covered code point is covered; bytes outside every haystack are False).  See
        _Automaton.mask_device."""
        self._ac.check_overlapping(overlapping)
        words = self._ac.mask_device(data, offsets, overlapping, flt=self._device_filter(data, offsets, pattern_sets, set_index))
        return self._ac.unpack_mask(words, data.numel())

    def count_matches_by_pattern(self, haystack: str, overlapping: bool = False) -> list:
        """-> list of length ``len(patterns)``: entry i is how many of ``find_matches_as_indexes(haystack,
        overlapping)`` have pattern i, counted without building the list."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.pattern_counts_host_batch([haystack.encode("utf-8")], overlapping)

    def count_matches_by_pattern_batch(self, haystacks: Sequence[str], overlapping: bool = False) -> list:
        """``count_matches_by_pattern`` summed over all the haystacks, in one transfer and one scan."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.pattern_counts_host_batch([h.encode("utf-8") for h in hays], overlapping)

    def count_matches_by_pattern_device(self, data, offsets, overlapping: bool = False):
        """Device-resident UTF-8 batch -> int64 tensor (n_patterns,) of match counts per pattern over the whole batch
        (see _Automaton.pattern_counts_device)."""
        return self._ac.pattern_counts_device(data, offsets, overlapping)

    # ---- additions: the patterns each haystack contains ---------------------------------------------------------
    def matching_patterns(self, haystack: str, overlapping: bool = False) -> list:
        """-> the distinct pattern ids of ``find_matches_as_indexes(haystack, overlapping)``, ascending, found without
        building the list."""
        if not isinstance(haystack, str):
            raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.hits_host_batch([haystack.encode("utf-8")], overlapping)[0]

    def matching_patterns_batch(self, haystacks: Sequence[str], overlapping: bool = False) -> list:
        """``matching_patterns`` for each haystack, in one transfer and one scan."""
        hays = list(haystacks)
        for h in hays:
            if not isinstance(h, str):
                raise TypeError("argument 'haystack': 'str' expected")
        self._ac.check_overlapping(overlapping)
        return self._ac.hits_host_batch([h.encode("utf-8") for h in hays], overlapping)

    def matching_patterns_device(self, data, offsets, overlapping: bool = False):
        """Device-resident UTF-8 batch -> (row_offsets, patterns, counts), the CSR form of each haystack's per-pattern
        match counts (see _Automaton.hits_device); the same in bytes and in code points."""
        return self._ac.hits_device(data, offsets, overlapping)

    # ---- additions: stream search (data fed in chunks; the crate's stream_find_iter, for every match kind) -------------
    def stream(self, overlapping: bool = False) -> Stream:
        """One stream fed ``str`` chunks: ``feed(chunk)`` returns the rows (pattern, start, end) it releases, in code
        points of the whole stream; ``finish()`` returns the rest.  All feeds together give
        ``find_matches_as_indexes(concatenation, overlapping)`` (see StreamBatch for when a row is released)."""
        self._ac.check_overlapping(overlapping)
        return Stream(self._ac, overlapping, codepoints=True)

    def stream_batch(self, n_streams: int, overlapping: bool = False) -> StreamBatch:
        """``n_streams`` streams fed from the device: ``feed_device(data, offsets, last=None)`` takes one UTF-8 chunk per
        stream (it may cut a character); positions are code point indexes (see StreamBatch)."""
        return StreamBatch(self._ac, n_streams, overlapping, codepoints=True)

    def is_match_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> IsMatchStreamBatch:
        """``n_streams`` is_match streams fed from the device: ``feed_device(data, offsets, last=None)`` -> bool CUDA
        tensor (n,), is_match of each stream's concatenation so far (see IsMatchStreamBatch).  pattern_sets= /
        set_index= (n_streams,): stream i searches only for the patterns of set set_index[i], for its whole life."""
        return _query_stream_batch(self._ac, "is_match", n_streams, False, codepoints=True, pattern_sets=pattern_sets, set_index=set_index)

    def find_first_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> FindFirstStreamBatch:
        """``n_streams`` find_first streams fed from the device: ``feed_device(data, offsets, last=None)`` -> int64 CUDA
        tensor (n, 3), each stream's first match once final, -1 rows while unknown (see FindFirstStreamBatch).
        pattern_sets= / set_index=: as for is_match_stream_batch."""
        return _query_stream_batch(self._ac, "find_first", n_streams, False, codepoints=True, pattern_sets=pattern_sets,
                                   set_index=set_index)

    def count_matches_stream_batch(self, n_streams: int, overlapping: bool = False) -> CountStreamBatch:
        """``n_streams`` count streams fed from the device: ``feed_device(data, offsets, last=None)`` -> int64 CUDA tensor
        (n,), the matches each stream's search has released so far (see CountStreamBatch)."""
        return _query_stream_batch(self._ac, "count", n_streams, overlapping, codepoints=True)

    def is_match_stream(self, patterns=None) -> QueryStream:
        """One is_match stream: ``feed(chunk)`` and ``finish()`` -> bool, does the concatenation so far contain a pattern
        (of `patterns`, when given)."""
        return _query_stream(self._ac, "is_match", False, codepoints=True, patterns=patterns)

    def find_first_stream(self, patterns=None) -> QueryStream:
        """One find_first stream: ``feed(chunk)`` and ``finish()`` -> (pattern, start, end) once no later data can change
        it, else None; ``finish()`` gives the final answer.  `patterns`: search only for these ids."""
        return _query_stream(self._ac, "find_first", False, codepoints=True, patterns=patterns)

    def count_matches_stream(self, overlapping: bool = False) -> QueryStream:
        """One count stream: ``feed(chunk)`` -> the matches released so far, ``finish()`` -> count_matches of the
        whole concatenation."""
        self._ac.check_overlapping(overlapping)
        return _query_stream(self._ac, "count", overlapping, codepoints=True)

    def match_mask_stream_batch(self, n_streams: int, overlapping: bool = False, pattern_sets=None, set_index=None) -> MaskStreamBatch:
        """``n_streams`` match-mask streams fed from the device: ``feed_device(data, offsets, last=None)`` -> (flags,
        flag_offsets, flag_starts), a flag per byte for each stream's bytes that no later data can change (see
        MaskStreamBatch).  pattern_sets= / set_index= (n_streams,): stream i searches only for set set_index[i]."""
        return _mask_stream_batch(self._ac, n_streams, overlapping, pattern_sets, set_index)

    def match_spans_stream(self, overlapping: bool = False, patterns=None) -> MaskStream:
        """One match-mask stream fed ``str`` chunks: ``feed(chunk)`` -> the runs (start, end) of covered code points
        this feed released, ``finish()`` -> the rest (see MaskStream).  `patterns`: search only for these ids."""
        return _mask_stream(self._ac, overlapping, True, patterns)

    def scan_host(self, data, offsets, overlapping: bool = False, **kw):
        """Host-resident UTF-8 batch (uint8 array + int64 offsets) -> host arrays (matches (k, 4), match_offsets (n + 1));
        code point indexes.  Copies and scans are pipelined (see _Automaton.scan_host)."""
        return self._ac.scan_host(data, offsets, overlapping, codepoints=True, **kw)


class BytesAhoCorasick(_PatternSetMethods):
    """Search for multiple pattern bytes against a bytes-like haystack
    (reference: src/lib.rs:342-363, 366-435).  No references to the patterns are kept."""

    def __init__(self, patterns: Iterable, matchkind: MatchKind = MatchKind.Standard,
                 implementation: Optional[Implementation] = None):
        if not isinstance(matchkind, MatchKind):
            raise TypeError("matchkind must be a MatchKind")
        if implementation is not None and not isinstance(implementation, Implementation):
            raise TypeError("implementation must be an Implementation or None")
        encoded = []
        for p in iter(patterns):
            b = _as_buffer_bytes(p)
            if len(b) == 0:
                raise ValueError("You passed in an empty pattern")
            encoded.append(b)
        self._ac = _Automaton(encoded, matchkind, implementation)

    def find_matches_as_indexes(self, haystack, overlapping: bool = False, patterns=None):
        """-> list of (pattern index, start, end) in byte offsets (src/lib.rs:422-434).  `patterns`: search only for
        these pattern ids (as an automaton of those patterns would; ids stay the full automaton's)."""
        hay = _as_buffer_bytes(haystack)
        self._ac.check_overlapping(overlapping)
        m, _ = self._ac.scan_host_batch([hay], overlapping, codepoints=False, patterns=_one_set(patterns))
        return _tuples(m)

    def find_matches_as_indexes_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None):
        self._ac.check_overlapping(overlapping)
        m, offs = self._ac.scan_host_batch([_as_buffer_bytes(h) for h in haystacks], overlapping, codepoints=False,
                                           patterns=_batch_sets(patterns, len(haystacks)))
        t = _tuples(m)
        return [t[offs[i]:offs[i + 1]] for i in range(len(haystacks))]

    def scan_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None, **kw):
        """Device-resident batch -> (matches, match_offsets, total); byte offsets.  pattern_sets= / set_index=:
        haystack i searches only for the patterns of set set_index[i]."""
        self._ac.check_overlapping(overlapping)
        return self._ac.scan_device(data, offsets, overlapping, codepoints=False,
                                    flt=self._device_filter(data, offsets, pattern_sets, set_index), **kw)

    # ---- additions: yes / no per haystack (the crate's AhoCorasick::is_match) ------------------------------
    def is_match(self, haystack, patterns=None) -> bool:
        """Does any pattern occur in `haystack` (a bytes-like object)?  The same for every match kind."""
        return self._ac.any_host_batch([_as_buffer_bytes(haystack)], _one_set(patterns))[0]

    def is_match_batch(self, haystacks: Sequence, patterns=None) -> list:
        """``is_match`` for each haystack, in one transfer and one scan."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        return self._ac.any_host_batch(hays, _batch_sets(patterns, len(hays)))

    def is_match_device(self, data, offsets, out=None, sync: bool = True, pattern_sets=None, set_index=None):
        """Device-resident batch -> bool tensor (n,) on its device (see _Automaton.any_device)."""
        return self._ac.any_device(data, offsets, out, sync, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: the first match per haystack (the crate's AhoCorasick::find) ---------------------------------
    def find_first(self, haystack, patterns=None):
        """-> (pattern index, start, end) in bytes, or None: ``find_matches_as_indexes(haystack)[0]``, found without
        the rest of the list."""
        return self._ac.first_host_batch([_as_buffer_bytes(haystack)], codepoints=False, patterns=_one_set(patterns))[0]

    def find_first_batch(self, haystacks: Sequence, patterns=None) -> list:
        """``find_first`` for each haystack, in one transfer and one scan."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        return self._ac.first_host_batch(hays, codepoints=False, patterns=_batch_sets(patterns, len(hays)))

    def find_first_device(self, data, offsets, pattern_sets=None, set_index=None):
        """Device-resident batch -> int64 tensor (n, 3) of (pattern, start, end) in bytes, -1 rows where a haystack has
        no match (see _Automaton.first_device)."""
        return self._ac.first_device(data, offsets, codepoints=False, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: match counts per haystack ------------------------------------------------------------------
    def count_matches(self, haystack, overlapping: bool = False, patterns=None) -> int:
        """-> ``len(find_matches_as_indexes(haystack, overlapping))``, counted without building the list."""
        hay = _as_buffer_bytes(haystack)
        self._ac.check_overlapping(overlapping)
        return self._ac.count_host_batch([hay], overlapping, _one_set(patterns))[0]

    def count_matches_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None) -> list:
        """``count_matches`` for each haystack, in one transfer and one scan."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        self._ac.check_overlapping(overlapping)
        return self._ac.count_host_batch(hays, overlapping, _batch_sets(patterns, len(hays)))

    def count_matches_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident batch -> int64 tensor (n,) of match counts (see _Automaton.count_device)."""
        self._ac.check_overlapping(overlapping)
        return self._ac.count_device(data, offsets, overlapping, flt=self._device_filter(data, offsets, pattern_sets, set_index))

    # ---- additions: which positions lie inside a match ---------------------------------------------------------
    def match_spans(self, haystack, overlapping: bool = False, patterns=None) -> list:
        """-> [(start, end), ...] in bytes: the maximal runs of bytes that lie inside some match of
        ``find_matches_as_indexes(haystack, overlapping)``.  Overlapping or touching matches merge into one span."""
        hay = _as_buffer_bytes(haystack)
        self._ac.check_overlapping(overlapping)
        return self._ac.spans_host_batch([hay], overlapping, False, _one_set(patterns))[0]

    def match_spans_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None) -> list:
        """``match_spans`` for each haystack, in one transfer and one scan; a span never crosses a haystack boundary."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        self._ac.check_overlapping(overlapping)
        return self._ac.spans_host_batch(hays, overlapping, False, _batch_sets(patterns, len(hays)))

    def match_mask_device(self, data, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident batch -> bool tensor of data's shape: byte p is True when it lies inside a match of its
        haystack (bytes outside every haystack are False).  See _Automaton.mask_device."""
        self._ac.check_overlapping(overlapping)
        words = self._ac.mask_device(data, offsets, overlapping, flt=self._device_filter(data, offsets, pattern_sets, set_index))
        return self._ac.unpack_mask(words, data.numel())

    def count_matches_by_pattern(self, haystack, overlapping: bool = False) -> list:
        """-> list of length ``len(patterns)``: entry i is how many of ``find_matches_as_indexes(haystack,
        overlapping)`` have pattern i, counted without building the list."""
        hay = _as_buffer_bytes(haystack)
        self._ac.check_overlapping(overlapping)
        return self._ac.pattern_counts_host_batch([hay], overlapping)

    def count_matches_by_pattern_batch(self, haystacks: Sequence, overlapping: bool = False) -> list:
        """``count_matches_by_pattern`` summed over all the haystacks, in one transfer and one scan."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        self._ac.check_overlapping(overlapping)
        return self._ac.pattern_counts_host_batch(hays, overlapping)

    def count_matches_by_pattern_device(self, data, offsets, overlapping: bool = False):
        """Device-resident batch -> int64 tensor (n_patterns,) of match counts per pattern over the whole batch (see
        _Automaton.pattern_counts_device)."""
        return self._ac.pattern_counts_device(data, offsets, overlapping)

    # ---- additions: the patterns each haystack contains ---------------------------------------------------------
    def matching_patterns(self, haystack, overlapping: bool = False) -> list:
        """-> the distinct pattern ids of ``find_matches_as_indexes(haystack, overlapping)``, ascending, found without
        building the list."""
        hay = _as_buffer_bytes(haystack)
        self._ac.check_overlapping(overlapping)
        return self._ac.hits_host_batch([hay], overlapping)[0]

    def matching_patterns_batch(self, haystacks: Sequence, overlapping: bool = False) -> list:
        """``matching_patterns`` for each haystack, in one transfer and one scan."""
        hays = [_as_buffer_bytes(h) for h in haystacks]
        self._ac.check_overlapping(overlapping)
        return self._ac.hits_host_batch(hays, overlapping)

    def matching_patterns_device(self, data, offsets, overlapping: bool = False):
        """Device-resident batch -> (row_offsets, patterns, counts), the CSR form of each haystack's per-pattern match
        counts (see _Automaton.hits_device)."""
        return self._ac.hits_device(data, offsets, overlapping)

    # ---- additions: stream search (data fed in chunks; the crate's stream_find_iter, for every match kind) -------------
    def stream(self, overlapping: bool = False) -> Stream:
        """One stream fed bytes-like chunks: ``feed(chunk)`` returns the rows (pattern, start, end) it releases, in byte
        offsets of the whole stream; ``finish()`` returns the rest.  All feeds together give
        ``find_matches_as_indexes(concatenation, overlapping)`` (see StreamBatch for when a row is released)."""
        self._ac.check_overlapping(overlapping)
        return Stream(self._ac, overlapping, codepoints=False)

    def stream_batch(self, n_streams: int, overlapping: bool = False) -> StreamBatch:
        """``n_streams`` streams fed from the device: ``feed_device(data, offsets, last=None)`` takes one chunk per
        stream; positions are byte offsets (see StreamBatch)."""
        return StreamBatch(self._ac, n_streams, overlapping, codepoints=False)

    def is_match_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> IsMatchStreamBatch:
        """``n_streams`` is_match streams fed from the device: ``feed_device(data, offsets, last=None)`` -> bool CUDA
        tensor (n,), is_match of each stream's concatenation so far (see IsMatchStreamBatch).  pattern_sets= /
        set_index= (n_streams,): stream i searches only for the patterns of set set_index[i], for its whole life."""
        return _query_stream_batch(self._ac, "is_match", n_streams, False, codepoints=False, pattern_sets=pattern_sets, set_index=set_index)

    def find_first_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> FindFirstStreamBatch:
        """``n_streams`` find_first streams fed from the device: ``feed_device(data, offsets, last=None)`` -> int64 CUDA
        tensor (n, 3), each stream's first match once final, -1 rows while unknown (see FindFirstStreamBatch).
        pattern_sets= / set_index=: as for is_match_stream_batch."""
        return _query_stream_batch(self._ac, "find_first", n_streams, False, codepoints=False, pattern_sets=pattern_sets,
                                   set_index=set_index)

    def count_matches_stream_batch(self, n_streams: int, overlapping: bool = False) -> CountStreamBatch:
        """``n_streams`` count streams fed from the device: ``feed_device(data, offsets, last=None)`` -> int64 CUDA tensor
        (n,), the matches each stream's search has released so far (see CountStreamBatch)."""
        return _query_stream_batch(self._ac, "count", n_streams, overlapping, codepoints=False)

    def is_match_stream(self, patterns=None) -> QueryStream:
        """One is_match stream: ``feed(chunk)`` and ``finish()`` -> bool, does the concatenation so far contain a pattern
        (of `patterns`, when given)."""
        return _query_stream(self._ac, "is_match", False, codepoints=False, patterns=patterns)

    def find_first_stream(self, patterns=None) -> QueryStream:
        """One find_first stream: ``feed(chunk)`` and ``finish()`` -> (pattern, start, end) once no later data can change
        it, else None; ``finish()`` gives the final answer.  `patterns`: search only for these ids."""
        return _query_stream(self._ac, "find_first", False, codepoints=False, patterns=patterns)

    def count_matches_stream(self, overlapping: bool = False) -> QueryStream:
        """One count stream: ``feed(chunk)`` -> the matches released so far, ``finish()`` -> count_matches of the
        whole concatenation."""
        self._ac.check_overlapping(overlapping)
        return _query_stream(self._ac, "count", overlapping, codepoints=False)

    def match_mask_stream_batch(self, n_streams: int, overlapping: bool = False, pattern_sets=None, set_index=None) -> MaskStreamBatch:
        """``n_streams`` match-mask streams fed from the device: ``feed_device(data, offsets, last=None)`` -> (flags,
        flag_offsets, flag_starts), a flag per byte for each stream's bytes that no later data can change (see
        MaskStreamBatch).  pattern_sets= / set_index= (n_streams,): stream i searches only for set set_index[i]."""
        return _mask_stream_batch(self._ac, n_streams, overlapping, pattern_sets, set_index)

    def match_spans_stream(self, overlapping: bool = False, patterns=None) -> MaskStream:
        """One match-mask stream fed bytes-like chunks: ``feed(chunk)`` -> the runs (start, end) of covered bytes this
        feed released, ``finish()`` -> the rest (see MaskStream).  `patterns`: search only for these ids."""
        return _mask_stream(self._ac, overlapping, False, patterns)

    def scan_host(self, data, offsets, overlapping: bool = False, **kw):
        """Host-resident batch (uint8 array + int64 offsets) -> host arrays (matches (k, 4), match_offsets (n + 1));
        byte offsets.  Copies and scans are pipelined (see _Automaton.scan_host)."""
        return self._ac.scan_host(data, offsets, overlapping, codepoints=False, **kw)


# ---- token ids: TokenAhoCorasick -------------------------------------------------------------------------------------
# Every id becomes ACB_TOKEN_BYTES bytes of a self-synchronising format (include/acb200.h, csrc/tokens.cuh: only a
# token's first byte has its high bit set), so a byte search over the encoded ids is exactly the token search with
# positions multiplied by 3.  Every query runs the byte path (codepoints=False) and divides the start and end columns.

_TOKEN_WIDTHS = (np.dtype(np.uint16), np.dtype(np.int32), np.dtype(np.int64))   # what acb_tokens_encode(_host) read


def _token_range_error(what: str, index: int, value) -> ValueError:
    return ValueError(f"{what}: token {index} = {value} is outside [0, {_capi.ACB_TOKEN_ID_LIMIT}) (ACB_TOKEN_ID_LIMIT)")


def _encode_host_tokens(seq, what: str) -> np.ndarray:
    """One 1-D integer sequence (list, tuple, numpy array or memmap, CPU tensor) -> its encoded bytes, a uint8 numpy
    array of 3 bytes per id (acb_tokens_encode_host).  TypeError for anything but integers, ValueError naming `what`,
    the index and the value of the first id outside [0, 2^21)."""
    a, ids = _host_token_ids(seq, what)
    if ids.size == 0:
        return np.zeros(0, dtype=np.uint8)
    out = np.empty(_capi.ACB_TOKEN_BYTES * ids.size, dtype=np.uint8)
    bad = np.full(1, np.iinfo(np.uint64).max, dtype=np.uint64)
    _check(_capi.lib().acb_tokens_encode_host(ids.ctypes.data, ids.itemsize, ids.size, out.ctypes.data, bad.ctypes.data))
    if bad[0] != np.iinfo(np.uint64).max:
        j = int(bad[0])
        raise _token_range_error(what, j, int(a[j]))
    return out


def _checked_host_ids(seq, what: str) -> np.ndarray:
    """One 1-D integer sequence -> its ids as a contiguous uint16 / int32 / int64 numpy array, with the errors of
    _encode_host_tokens (the range checked here, without encoding)."""
    a, ids = _host_token_ids(seq, what)
    bad = np.flatnonzero((ids < 0) | (ids >= _capi.ACB_TOKEN_ID_LIMIT))
    if bad.size:
        j = int(bad[0])
        raise _token_range_error(what, j, int(a[j]))
    return ids


def _host_token_ids(seq, what: str):
    """The type checks of _encode_host_tokens -> (the sequence as a numpy array, its ids as a contiguous uint16 /
    int32 / int64 array; empty for an empty sequence).  Ids of object arrays are range-checked here, the rest not."""
    torch = __import__("sys").modules.get("torch")
    if torch is not None and torch.is_tensor(seq):
        if seq.device.type != "cpu":
            raise TypeError(f"{what}: a CUDA tensor goes to the *_device methods; this form takes host sequences")
        seq = seq.detach().numpy()
    try:
        a = np.asarray(seq)
    except ValueError as e:   # ragged nesting
        raise TypeError(f"{what} must be a one-dimensional sequence of token ids") from e
    if a.ndim != 1:
        raise TypeError(f"{what} must be a one-dimensional sequence of token ids")
    if a.size == 0:
        return a, np.zeros(0, dtype=np.int64)
    if a.dtype == object:   # Python ints beyond int64, or mixed objects
        for j, v in enumerate(a.tolist()):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise TypeError(f"{what}: token ids must be integers, not {type(v).__name__}")
            if not 0 <= v < _capi.ACB_TOKEN_ID_LIMIT:
                raise _token_range_error(what, j, v)
        ids = np.asarray(a.tolist(), dtype=np.int64)
    elif a.dtype.kind not in "iu":
        raise TypeError(f"{what}: token ids must be integers, not {a.dtype}")
    elif a.dtype in _TOKEN_WIDTHS:
        ids = np.ascontiguousarray(a)
    else:   # narrower ints widen to int32, uint32 / uint64 to int64 (an id past 2^63 wraps negative: still out of range)
        ids = np.ascontiguousarray(a, dtype=np.int32 if a.itemsize < 4 else np.int64)
    return a, ids


def _token_offsets(offsets, tokens):
    """Token offsets -> byte offsets (x 3).  They must lie in [0, len(tokens)] (one synchronisation): a larger or
    negative offset would wrap in the multiplication and could put a haystack boundary inside a token."""
    torch = _torch()
    if not torch.is_tensor(offsets) or offsets.dtype != torch.int64:
        raise TypeError("offsets must be an int64 tensor of token offsets")
    if torch.is_tensor(tokens) and offsets.numel():
        n = tokens.numel()
        if bool(((offsets < 0) | (offsets > n)).any().item()):
            raise ValueError(f"offsets must lie in [0, {n}] (token offsets into the {n} ids)")
    return offsets * _capi.ACB_TOKEN_BYTES


def _token_rows(m, cols):
    """A new tensor: the byte search's rows with their position columns `cols` (a slice) divided by 3.  Floor division
    keeps the -1 of a row without a match at -1."""
    out = m.clone()
    out[:, cols] //= _capi.ACB_TOKEN_BYTES
    return out


class _TokenEncoder:
    """acb_tokens_encode into one grow-only byte buffer per device.  Callers hold `lock` from the encode until every
    scan that reads the buffer has been enqueued, then call done(): the next encode waits, on its own stream, for
    those scans (a query that returns before its scan has finished may still be reading the buffer)."""

    def __init__(self):
        self.lock = threading.RLock()
        self._bufs = {}      # device index -> uint8 tensor
        self._readers = {}   # device index -> CUDA event after the last scan of the buffer

    def encode(self, tokens):
        """A 1-D uint16 / int32 / int64 CUDA tensor of ids -> a uint8 view of the buffer holding their bytes.  An id
        outside [0, 2^21) raises ValueError with its index and value (the call waits for the kernel to know)."""
        torch = _require_cuda()
        if (not torch.is_tensor(tokens) or tokens.dim() != 1 or tokens.device.type != "cuda" or
                tokens.dtype not in (torch.uint16, torch.int32, torch.int64)):
            raise TypeError("tokens must be a 1-D CUDA tensor of uint16, int32 or int64 token ids")
        tokens = tokens.contiguous()
        dev = tokens.device
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        n = tokens.numel()
        nbytes = _capi.ACB_TOKEN_BYTES * n
        stream = torch.cuda.current_stream(dev)
        reader = self._readers.get(idx)   # (dropped only once this encode is enqueued behind it)
        buf = self._bufs.get(idx)
        if buf is None or buf.numel() < nbytes:
            if reader is not None:
                reader.synchronize()   # the old buffer goes back to the allocator: no scan may still read it
            buf = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, device=dev)
            self._bufs[idx] = buf
        elif reader is not None:
            stream.wait_event(reader)
        bad = torch.full((1,), -1, dtype=torch.int64, device=dev)   # ~0: no bad id
        with torch.cuda.device(dev):
            rc = _capi.lib().acb_tokens_encode(tokens.data_ptr(), tokens.element_size(), n, buf.data_ptr(), bad.data_ptr(),
                                               stream.cuda_stream)
        _check(rc)
        self._readers.pop(idx, None)
        j = int(bad.item())
        if j != -1:
            raise _token_range_error("tokens", j, int(tokens[j].item()))
        return buf[:nbytes]

    def done(self, dev):
        torch = _torch()
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        self._readers[idx] = ev


def _token_stream_limits(ac: "_Automaton", n_streams):
    """The stream limits of StreamBatch, stated in tokens: the seams of one feed (2 x (max_pattern_len - 1) bytes per
    stream) must fit WINDOW_BYTES.  Arguments StreamBatch refuses on their own are left to it."""
    if isinstance(n_streams, bool) or not isinstance(n_streams, int) or n_streams < 0:
        return
    k = ac.max_pattern_len // _capi.ACB_TOKEN_BYTES
    seam = 2 * n_streams * max(ac.max_pattern_len - 1, 0)
    if seam > ac.WINDOW_BYTES:
        raise ValueError(f"{n_streams} streams x 2 x (3 x {k} - 1) = {seam} seam bytes, with the longest pattern at {k} tokens: one "
                         f"feed's seams must fit {ac.WINDOW_BYTES} bytes (WINDOW_BYTES); use fewer streams per batch")


def _token_feed_limit(ac: "_Automaton", n_tokens: int):
    limit = ac.WINDOW_BYTES // _capi.ACB_TOKEN_BYTES
    if n_tokens > limit:
        raise ValueError(f"one feed addresses at most {limit} tokens (WINDOW_BYTES / 3): feed larger data in more chunks")


class TokenStreamBatch:
    """A StreamBatch or a stream query batch over token ids: feed_device(tokens, offsets, last=None) takes one chunk of
    ids per stream (a 1-D uint16 / int32 / int64 CUDA tensor, int64 offsets (n_streams + 1) in tokens) and returns
    what the wrapped batch returns, positions in tokens: (rows (k, 4), row_offsets) for stream_batch, the answers for
    the query batches."""

    def __init__(self, batch, convert):
        self._batch = batch
        self._convert = convert
        self._enc = _TokenEncoder()

    n_streams = property(lambda self: self._batch.n_streams)
    overlapping = property(lambda self: self._batch.overlapping)
    device = property(lambda self: self._batch.device)
    last_stats = property(lambda self: self._batch.last_stats)

    def feed_device(self, tokens, offsets, last=None):
        _require_cuda()
        if _torch().is_tensor(tokens):
            _token_feed_limit(self._batch._ac, tokens.numel())
        offsets = _token_offsets(offsets, tokens)
        # the wrapped feed_device reads the encoded chunk in place and synchronises before it returns (it reads its
        # row counts), so the next feed may encode into the same buffer
        with self._enc.lock:
            data = self._enc.encode(tokens)
            return self._convert(self._batch.feed_device(data, offsets, last))


class TokenStream:
    """A Stream or a query stream fed host chunks of token ids (1-D integer sequences): feed(chunk) and finish() return
    what the wrapped stream returns, positions in tokens."""

    def __init__(self, stream, convert):
        self._stream = stream
        self._convert = convert

    last_stats = property(lambda self: self._stream.last_stats)

    def feed(self, chunk):
        data = _encode_host_tokens(chunk, "chunk")
        _token_feed_limit(self._stream._batch._ac, data.size // _capi.ACB_TOKEN_BYTES)
        return self._convert(self._stream._feed(data, False))

    def finish(self):
        return self._convert(self._stream._feed(b"", True))


class TokenMaskStream(TokenStream):
    """A MaskStream fed host chunks of token ids; `released` counts tokens."""

    released = property(lambda self: self._stream.released)


def _same(x):
    return x


def _token_first_answer(row):
    return (row[0], row[1] // _capi.ACB_TOKEN_BYTES, row[2] // _capi.ACB_TOKEN_BYTES) if row[0] >= 0 else None


def _token_tuples(m: np.ndarray):
    return list(zip(m[:, 1].tolist(), (m[:, 2] // _capi.ACB_TOKEN_BYTES).tolist(), (m[:, 3] // _capi.ACB_TOKEN_BYTES).tolist()))


class TokenAhoCorasick(_PatternSetMethods):
    """Search for multiple token-id sequences against token-id sequences: tokenized corpora (uint16 / int32 arrays),
    generation outputs (int64 tensors).  Positions are token indexes; everything else is BytesAhoCorasick's.

    * ``patterns``: an iterable of non-empty 1-D integer sequences (lists, tuples, numpy arrays, CPU tensors) of ids
      in [0, 2^21) (ACB_TOKEN_ID_LIMIT).
    * ``matchkind``, ``implementation``: as for BytesAhoCorasick.

    The ids are encoded into a self-synchronising 3-byte format (include/acb200.h) and searched by the byte engine:
    host forms encode on the host, device forms with acb_tokens_encode into a grow-only buffer per device.
    ``max_pattern_len`` is in bytes (3 x the longest pattern's tokens)."""

    def __init__(self, patterns: Iterable, matchkind: MatchKind = MatchKind.Standard,
                 implementation: Optional[Implementation] = None):
        if not isinstance(matchkind, MatchKind):
            raise TypeError("matchkind must be a MatchKind")
        if implementation is not None and not isinstance(implementation, Implementation):
            raise TypeError("implementation must be an Implementation or None")
        encoded = []
        for i, p in enumerate(iter(patterns)):
            b = _encode_host_tokens(p, f"pattern {i}")
            if b.size == 0:
                raise ValueError("You passed in an empty pattern")
            encoded.append(b.tobytes())
        self._ac = _Automaton(encoded, matchkind, implementation)
        self._enc = _TokenEncoder()

    @property
    def max_pattern_len(self) -> int:
        return self._ac.max_pattern_len

    @property
    def last_stats(self):
        return self._ac.last_stats

    def _hays(self, haystacks):
        return [_encode_host_tokens(h, f"haystack {i}") for i, h in enumerate(haystacks)]

    def _on_device(self, query, tokens, offsets):
        """query(data, byte offsets) on the encoded ids of a device batch, the encode buffer guarded until it is read."""
        torch = _torch()
        offsets = _token_offsets(offsets, tokens)
        with self._enc.lock:
            data = self._enc.encode(tokens)
            with torch.cuda.device(data.device):
                out = query(data, offsets)
                self._enc.done(data.device)
        return out

    # ---- the match list ----------------------------------------------------------------------------------------------
    def _token_filter(self, tokens, offsets, pattern_sets, set_index):
        if pattern_sets is None and set_index is None:
            return None
        n = (offsets.numel() if hasattr(offsets, "numel") else len(offsets)) - 1
        return _filter_args(self._ac, pattern_sets, set_index, n, tokens.device if hasattr(tokens, "device") else None)

    def find_matches_as_indexes(self, haystack, overlapping: bool = False, patterns=None):
        """-> list of (pattern index, start, end) in token indexes.  `patterns`: search only for these pattern ids."""
        hay = _encode_host_tokens(haystack, "haystack")
        self._ac.check_overlapping(overlapping)
        m, _ = self._ac.scan_host_batch([hay], overlapping, codepoints=False, patterns=_one_set(patterns))
        return _token_tuples(m)

    def find_matches_as_indexes_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None):
        """One list of (pattern, start, end) per haystack, each what ``find_matches_as_indexes`` returns for it."""
        hays = self._hays(haystacks)
        self._ac.check_overlapping(overlapping)
        m, offs = self._ac.scan_host_batch(hays, overlapping, codepoints=False, patterns=_batch_sets(patterns, len(hays)))
        t = _token_tuples(m)
        return [t[offs[i]:offs[i + 1]] for i in range(len(hays))]

    def scan_device(self, tokens, offsets, overlapping: bool = False, capacity: Optional[int] = None, pattern_sets=None, set_index=None):
        """Device-resident batch of ids (1-D uint16 / int32 / int64 CUDA tensor, int64 offsets (n + 1) in tokens) ->
        (matches, match_offsets, total) as BytesAhoCorasick.scan_device returns them (int32 rows, int64 above
        WINDOW_BYTES encoded bytes), positions in tokens.  The tensors are the caller's own, not workspace views."""
        self._ac.check_overlapping(overlapping)
        torch = _torch()
        flt = self._token_filter(tokens, offsets, pattern_sets, set_index)

        def query(data, offs):
            # the automaton's scan_device returns views of its workspace slot 0: the copies are enqueued under its
            # lock, and the next scan on that slot (any thread, any stream) waits for them, as first_device's gather
            with self._ac._lock:
                m, mo, total = self._ac.scan_device(data, offs, overlapping, codepoints=False, capacity=capacity, flt=flt)
                out = _token_rows(m, slice(2, 4)), mo.clone(), total
                self._ac._mark_read(data.device)
            return out
        return self._on_device(query, tokens, offsets)

    # ---- queries -----------------------------------------------------------------------------------------------------
    def is_match(self, haystack, patterns=None) -> bool:
        """Does any pattern occur in `haystack`?  The same for every match kind."""
        return self._ac.any_host_batch(self._hays([haystack]), _one_set(patterns))[0]

    def is_match_batch(self, haystacks: Sequence, patterns=None) -> list:
        hays = self._hays(haystacks)
        return self._ac.any_host_batch(hays, _batch_sets(patterns, len(hays)))

    def is_match_device(self, tokens, offsets, pattern_sets=None, set_index=None):
        """Device-resident batch of ids -> bool tensor (n,) (see _Automaton.any_device)."""
        flt = self._token_filter(tokens, offsets, pattern_sets, set_index)
        return self._on_device(lambda d, o: self._ac.any_device(d, o, flt=flt), tokens, offsets)

    def find_first(self, haystack, patterns=None):
        """-> (pattern index, start, end) in token indexes, or None: ``find_matches_as_indexes(haystack)[0]``."""
        return self.find_first_batch([haystack], _one_set(patterns))[0]

    def find_first_batch(self, haystacks: Sequence, patterns=None) -> list:
        hays = self._hays(haystacks)
        rows = self._ac.first_host_batch(hays, codepoints=False, patterns=_batch_sets(patterns, len(hays)))
        return [_token_first_answer(r) if r is not None else None for r in rows]

    def find_first_device(self, tokens, offsets, pattern_sets=None, set_index=None):
        """Device-resident batch of ids -> int64 tensor (n, 3) of (pattern, start, end) in tokens, -1 rows where a
        haystack has no match (see _Automaton.first_device)."""
        flt = self._token_filter(tokens, offsets, pattern_sets, set_index)
        return self._on_device(lambda d, o: _token_rows(self._ac.first_device(d, o, flt=flt), slice(1, 3)), tokens, offsets)

    def count_matches(self, haystack, overlapping: bool = False, patterns=None) -> int:
        """-> ``len(find_matches_as_indexes(haystack, overlapping))``, counted without building the list."""
        return self.count_matches_batch([haystack], overlapping, _one_set(patterns))[0]

    def count_matches_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None) -> list:
        hays = self._hays(haystacks)
        self._ac.check_overlapping(overlapping)
        return self._ac.count_host_batch(hays, overlapping, _batch_sets(patterns, len(hays)))

    def count_matches_device(self, tokens, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident batch of ids -> int64 tensor (n,) of match counts (see _Automaton.count_device)."""
        self._ac.check_overlapping(overlapping)
        flt = self._token_filter(tokens, offsets, pattern_sets, set_index)
        return self._on_device(lambda d, o: self._ac.count_device(d, o, overlapping, flt=flt), tokens, offsets)

    def match_spans(self, haystack, overlapping: bool = False, patterns=None) -> list:
        """-> [(start, end), ...] in tokens: the maximal runs of tokens that lie inside some match of
        ``find_matches_as_indexes(haystack, overlapping)``."""
        return self.match_spans_batch([haystack], overlapping, _one_set(patterns))[0]

    def match_spans_batch(self, haystacks: Sequence, overlapping: bool = False, patterns=None) -> list:
        hays = self._hays(haystacks)
        self._ac.check_overlapping(overlapping)
        return self._ac.spans_host_batch(hays, overlapping, False, _batch_sets(patterns, len(hays)), unit=_capi.ACB_TOKEN_BYTES)

    def match_mask_device(self, tokens, offsets, overlapping: bool = False, pattern_sets=None, set_index=None):
        """Device-resident batch of ids -> bool tensor (len(tokens),): token i is True when it lies inside a match of its
        haystack (a per-token loss mask of banned sequences).  The mask is built over the encoded bytes and read at
        every token's first byte: an occurrence starts and ends on a token boundary."""
        self._ac.check_overlapping(overlapping)
        flt = self._token_filter(tokens, offsets, pattern_sets, set_index)
        n = tokens.numel() if hasattr(tokens, "numel") else 0
        return self._on_device(lambda d, o: self._ac.unpack_mask(self._ac.mask_device(d, o, overlapping, flt=flt), n, _capi.ACB_TOKEN_BYTES),
                               tokens, offsets)

    def count_matches_by_pattern(self, haystack, overlapping: bool = False) -> list:
        """-> entry i is how many of ``find_matches_as_indexes(haystack, overlapping)`` have pattern i."""
        return self.count_matches_by_pattern_batch([haystack], overlapping)

    def count_matches_by_pattern_batch(self, haystacks: Sequence, overlapping: bool = False) -> list:
        hays = self._hays(haystacks)
        self._ac.check_overlapping(overlapping)
        return self._ac.pattern_counts_host_batch(hays, overlapping)

    def count_matches_by_pattern_device(self, tokens, offsets, overlapping: bool = False):
        """Device-resident batch of ids -> int64 tensor (n_patterns,) (see _Automaton.pattern_counts_device)."""
        self._ac.check_overlapping(overlapping)
        return self._on_device(lambda d, o: self._ac.pattern_counts_device(d, o, overlapping), tokens, offsets)

    def matching_patterns(self, haystack, overlapping: bool = False) -> list:
        """-> the distinct pattern ids of ``find_matches_as_indexes(haystack, overlapping)``, ascending."""
        return self.matching_patterns_batch([haystack], overlapping)[0]

    def matching_patterns_batch(self, haystacks: Sequence, overlapping: bool = False) -> list:
        hays = self._hays(haystacks)
        self._ac.check_overlapping(overlapping)
        return self._ac.hits_host_batch(hays, overlapping)

    def matching_patterns_device(self, tokens, offsets, overlapping: bool = False):
        """Device-resident batch of ids -> (row_offsets, patterns, counts) (see _Automaton.hits_device)."""
        self._ac.check_overlapping(overlapping)
        return self._on_device(lambda d, o: self._ac.hits_device(d, o, overlapping), tokens, offsets)

    # ---- completing tokens: the next ids that would complete a pattern -----------------------------------------------
    # Id t completes a pattern for a row with history C when some admitted pattern p is a suffix of C || [t]: p[:-1] is
    # a suffix of C and p[-1] == t (a match of a Standard search would end right after C).  It does not depend on the
    # match kind, and only the last K - 1 ids of C matter (K = the longest pattern in tokens).  One warp per row walks
    # the completions image (csrc/completions.h) backwards over those ids (include/acb200.h, acb_completions_*).
    def _completions_args(self, tokens, offsets, pattern_sets, set_index):
        """The device forms' checks, none of which reads the device: -> (tokens, offsets, n, filter)."""
        torch = _torch()
        if (not torch.is_tensor(tokens) or tokens.dim() != 1 or tokens.device.type != "cuda" or
                tokens.dtype not in (torch.uint16, torch.int32, torch.int64)):
            raise TypeError("tokens must be a 1-D CUDA tensor of uint16, int32 or int64 token ids")
        if not torch.is_tensor(offsets) or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1:
            raise TypeError("offsets must be a 1-D int64 tensor of n + 1 token offsets")
        if offsets.device != tokens.device:
            raise ValueError(f"offsets live on {offsets.device}, the tokens on {tokens.device}")
        n = offsets.numel() - 1
        flt = _filter_shape_args(self._ac, pattern_sets, set_index, n, tokens.device)
        _require_cuda()
        return tokens.contiguous(), offsets.contiguous(), n, flt

    def _completions_stats(self, desc):
        self._ac.last_stats = {"mode": "completions", "nodes": int(desc.nodes), "entries": int(desc.entries)}

    def completing_tokens(self, history, patterns=None) -> list:
        """-> the sorted distinct ids t for which some pattern (of `patterns`, when given) is a suffix of
        ``history + [t]``: the next tokens that would complete a pattern.  Ids outside [0, 2^21) raise ValueError."""
        return self.completing_tokens_batch([history], _one_set(patterns))[0]

    def completing_tokens_batch(self, histories: Sequence, patterns=None) -> list:
        """One sorted list of completing ids per history (``completing_tokens`` of each); `patterns`: one iterable of
        pattern ids per history.  The last K - 1 ids of every history go to the device in one batch."""
        hists = [_checked_host_ids(h, f"history {i}") for i, h in enumerate(histories)]
        n = len(hists)
        sets = _batch_sets(patterns, n)
        if n == 0:
            return []
        torch = _require_cuda()
        dev = torch.device("cuda", torch.cuda.current_device())
        depth = int(self._ac.completions(dev)[1].depth)
        tails = [ids[max(ids.size - depth, 0):].astype(np.int64) for ids in hists]
        flt = None if sets is None else _host_sets(self._ac, sets, n, dev)
        offs = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([t.size for t in tails], out=offs[1:])
        tokens = torch.from_numpy(np.concatenate(tails)).to(dev)
        with torch.cuda.device(dev):
            ids, row_offsets = self._completions_csr(tokens, torch.from_numpy(offs).to(dev), n, flt)
        ids, row_offsets = ids.cpu().numpy(), row_offsets.cpu().numpy()
        return [ids[row_offsets[i]:row_offsets[i + 1]].tolist() for i in range(n)]

    def completing_tokens_device(self, tokens, offsets, pattern_sets=None, set_index=None):
        """Device-resident histories -> (ids int64 (k,), row_offsets int64 (n + 1,)): row i's completing ids are
        ids[row_offsets[i]:row_offsets[i + 1]], ascending and distinct.  One synchronisation (k).

        ``tokens``: a 1-D uint16 / int32 / int64 CUDA tensor; ``offsets``: int64 (n + 1,) in tokens.  An (n, L)
        ``input_ids`` tensor is passed as ``ids.reshape(-1)`` with ``offsets = arange(n + 1) * L``.  Offsets are not
        validated: row i's history is tokens[a:b], a and b being offsets[i] and offsets[i + 1] clamped to
        [0, len(tokens)], and b < a is an empty history.  Ids outside [0, 2^21) (a negative pad id) equal no pattern
        token.  ``pattern_sets`` / ``set_index`` (n,): each row's own set; an index outside [0, n_sets) admits nothing."""
        tokens, offsets, n, flt = self._completions_args(tokens, offsets, pattern_sets, set_index)
        torch = _torch()
        with torch.cuda.device(tokens.device):
            return self._completions_csr(tokens, offsets, n, flt)

    def _completions_csr(self, tokens, offsets, n: int, flt):
        torch = _torch()
        dev = tokens.device
        img, desc = self._ac.completions(dev)
        L = self._ac._L
        st = torch.cuda.current_stream(dev).cuda_stream
        counts = torch.empty(n, dtype=torch.int64, device=dev)
        _check(L.acb_completions_count(self._ac._h, img.data_ptr(), tokens.data_ptr(), tokens.element_size(), tokens.numel(),
                                       offsets.data_ptr(), n, counts.data_ptr(), _filter_struct(flt), st))
        row_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=row_offsets[1:])
        k = int(row_offsets[-1].item())
        ids = torch.empty(k, dtype=torch.int64, device=dev)
        if k:
            _check(L.acb_completions_emit(self._ac._h, img.data_ptr(), tokens.data_ptr(), tokens.element_size(), tokens.numel(),
                                          offsets.data_ptr(), n, row_offsets.data_ptr(), ids.data_ptr(), _filter_struct(flt), st))
            # each row's ids come out distinct and ascending per trie node: one sort of (row, id) keys orders them
            rows = torch.repeat_interleave(torch.arange(n, device=dev), counts, output_size=k)
            ids = torch.bitwise_and(torch.sort(rows * _capi.ACB_TOKEN_ID_LIMIT + ids).values, _capi.ACB_TOKEN_ID_LIMIT - 1)
        self._completions_stats(desc)
        return ids, row_offsets

    _LOGITS_DTYPES = {"float32": _capi.ACB_LOGITS_F32, "float16": _capi.ACB_LOGITS_F16, "bfloat16": _capi.ACB_LOGITS_BF16}

    def mask_completing_tokens_(self, logits, tokens, offsets, pattern_sets=None, set_index=None, value: float = float("-inf")):
        """In place: logits[i, t] = value for every id t that completes a pattern for row i (the bad-words logits
        processor: ban every next token that would finish a banned sequence); every other element is untouched.
        Returns `logits`.

        ``logits``: float32 / float16 / bfloat16 CUDA tensor (n, V) with stride(1) == 1 and any row stride (so
        ``scores[:, -1, :]`` works).  ``tokens``, ``offsets``, ``pattern_sets``, ``set_index``: as for
        ``completing_tokens_device`` -- an (n, L) ``input_ids`` tensor is ``ids.reshape(-1)`` with
        ``offsets = arange(n + 1) * L``; offsets are clamped to [0, len(tokens)], not validated; a set index outside
        [0, n_sets) bans nothing.  Nothing is read back and, for contiguous tokens, offsets and set_index, nothing is
        allocated: after the first call (which builds and uploads the image) the call can be captured in a CUDA graph.
        ValueError when the largest id that ends a pattern is >= V (checked on the host)."""
        tokens, offsets, n, flt = self._completions_args(tokens, offsets, pattern_sets, set_index)
        torch = _torch()
        code, V, img, desc = self._logits_args(logits, tokens, n)
        with torch.cuda.device(tokens.device):
            rc = self._ac._L.acb_completions_mask(self._ac._h, img.data_ptr(), tokens.data_ptr(), tokens.element_size(), tokens.numel(),
                                                  offsets.data_ptr(), n, logits.data_ptr(), code, logits.stride(0) if n > 1 else V, V,
                                                  float(value), _filter_struct(flt), torch.cuda.current_stream(tokens.device).cuda_stream)
        _check(rc)
        self._completions_stats(desc)
        return logits

    def _logits_args(self, logits, tokens, n: int):
        """The logits checks of the mask and the bias, none of which reads the device, and the vocabulary check against
        the image's largest last id (on the host): -> (dtype code, V, image, desc)."""
        torch = _torch()
        code = self._LOGITS_DTYPES.get(str(logits.dtype).replace("torch.", "")) if torch.is_tensor(logits) else None
        if code is None or logits.dim() != 2:
            raise TypeError("logits must be a 2-D float32, float16 or bfloat16 tensor (n, V)")
        if logits.device != tokens.device:
            raise ValueError(f"logits live on {logits.device}, the tokens on {tokens.device}")
        V = int(logits.shape[1])
        if logits.shape[0] != n:
            raise ValueError(f"logits have {logits.shape[0]} rows, offsets describe {n} histories")
        if V < 1:
            raise ValueError("logits need at least one column")
        if logits.stride(1) != 1 and V > 1:
            raise ValueError("logits rows must be contiguous (stride(1) == 1); any row stride is fine")
        img, desc = self._ac.completions(tokens.device)
        if desc.entries and desc.max_last >= V:
            raise ValueError(f"logits have {V} columns, but id {desc.max_last} ends a pattern: V must exceed every pattern's last id")
        return code, V, img, desc

    def bias_completing_tokens_(self, logits, tokens, offsets, bias, pattern_sets=None, set_index=None):
        """In place: adds a signed bias per pattern to the ids that would complete it (the sequence-bias logits
        processor: a positive bias encourages a sequence, a negative one discourages it, -inf bans it).  Returns
        `logits`.

        ``bias``: float32 CUDA tensor (len(patterns),) on the tokens' device.  For row i and id t, let P_t be the
        admitted pids p that t completes (p[:-1] is a suffix of the row's history and p[-1] == t), ordered longest
        pattern first, ties by ascending pid: s = bias[p1] + bias[p2] + ... summed in float32 from the first term, then
        logits[i, t] = logits[i, t] + s computed in float32 and rounded once (nearest-even) to the logits dtype.
        Every other element is untouched, and the result is the same bit for bit on every run.  With every bias -inf
        this equals ``mask_completing_tokens_``.  Per-request values: give the same sequence twice, as two patterns
        with their own biases, each in its request's pattern set; duplicates that are both admitted both count.

        Differences from Hugging Face's ``SequenceBiasLogitsProcessor``: it accumulates in the logits dtype, in dict
        order, where this sums in float32 and rounds once; and it skips every sequence longer than the padded batch
        width and compares pad ids, where this applies every pattern whose p[:-1] is a suffix of the row's own history.

        ``logits``, ``tokens``, ``offsets``, ``pattern_sets``, ``set_index``: as for ``mask_completing_tokens_``.
        Nothing is read back and, for contiguous inputs, nothing is allocated: after the first call the call can be
        captured in a CUDA graph (rewrite the histories, set indices and biases in place between replays)."""
        tokens, offsets, n, flt = self._completions_args(tokens, offsets, pattern_sets, set_index)
        torch = _torch()
        P = self._ac.n_patterns
        if not torch.is_tensor(bias) or bias.dtype != torch.float32:
            raise TypeError("bias must be a float32 tensor with one value per pattern")
        if bias.dim() != 1 or bias.numel() != P:
            raise ValueError(f"bias has shape {tuple(bias.shape)}, expected ({P},): one value per pattern")
        if bias.device != tokens.device:
            raise ValueError(f"bias lives on {bias.device}, the tokens on {tokens.device}")
        code, V, img, desc = self._logits_args(logits, tokens, n)
        if P:   # without patterns there is nothing to add (and an empty bias has no storage to pass)
            bias = bias.contiguous()
            with torch.cuda.device(tokens.device):
                rc = self._ac._L.acb_completions_bias(self._ac._h, img.data_ptr(), tokens.data_ptr(), tokens.element_size(),
                                                      tokens.numel(), offsets.data_ptr(), n, bias.data_ptr(), logits.data_ptr(), code,
                                                      logits.stride(0) if n > 1 else V, V, _filter_struct(flt),
                                                      torch.cuda.current_stream(tokens.device).cuda_stream)
            _check(rc)
        self._completions_stats(desc)
        return logits

    # ---- streams: ids fed in chunks ----------------------------------------------------------------------------------
    def stream(self, overlapping: bool = False) -> TokenStream:
        """One stream fed host chunks of ids: ``feed(chunk)`` returns the rows (pattern, start, end) it releases, in
        tokens of the whole stream; ``finish()`` returns the rest (see StreamBatch)."""
        self._ac.check_overlapping(overlapping)
        _token_stream_limits(self._ac, 1)
        return TokenStream(Stream(self._ac, overlapping, codepoints=False), _token_tuples_of_rows)

    def stream_batch(self, n_streams: int, overlapping: bool = False) -> TokenStreamBatch:
        """``n_streams`` streams fed from the device: ``feed_device(tokens, offsets, last=None)`` -> (rows (k, 4) int64,
        row_offsets), positions in tokens (see StreamBatch)."""
        _token_stream_limits(self._ac, n_streams)
        return TokenStreamBatch(StreamBatch(self._ac, n_streams, overlapping, codepoints=False),
                                lambda r: (_token_rows(r[0], slice(2, 4)), r[1]))

    def _query_batch(self, kind, n_streams, overlapping, pattern_sets=None, set_index=None):
        _token_stream_limits(self._ac, n_streams)
        convert = (lambda rows: _token_rows(rows, slice(1, 3))) if kind == "find_first" else _same
        return TokenStreamBatch(_query_stream_batch(self._ac, kind, n_streams, overlapping, codepoints=False, pattern_sets=pattern_sets,
                                                    set_index=set_index), convert)

    def _query_stream(self, kind, overlapping, patterns=None):
        _token_stream_limits(self._ac, 1)
        answer = {"is_match": bool, "find_first": _token_first_answer, "count": int}[kind]
        if patterns is None:
            return TokenStream(QueryStream(_query_stream_batch(self._ac, kind, 1, overlapping, codepoints=False), answer), _same)
        torch = _require_cuda()
        ps = self.pattern_sets([patterns])
        batch = _query_stream_batch(self._ac, kind, 1, overlapping, codepoints=False, pattern_sets=ps,
                                    set_index=torch.zeros(1, dtype=torch.int32, device=ps.device))
        return TokenStream(QueryStream(batch, answer), _same)

    def is_match_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> TokenStreamBatch:
        """``feed_device`` -> bool CUDA tensor (n,), is_match of each stream so far (see IsMatchStreamBatch);
        pattern_sets= / set_index= (n_streams,) fix each stream's pattern set."""
        return self._query_batch("is_match", n_streams, False, pattern_sets, set_index)

    def find_first_stream_batch(self, n_streams: int, pattern_sets=None, set_index=None) -> TokenStreamBatch:
        """``feed_device`` -> int64 CUDA tensor (n, 3), each stream's first match in tokens once final, -1 rows while
        unknown (see FindFirstStreamBatch); pattern_sets= / set_index= (n_streams,) fix each stream's pattern set
        (per-request stop sequences in batched generation)."""
        return self._query_batch("find_first", n_streams, False, pattern_sets, set_index)

    def count_matches_stream_batch(self, n_streams: int, overlapping: bool = False) -> TokenStreamBatch:
        """``feed_device`` -> int64 CUDA tensor (n,), the matches each stream's search has released (see CountStreamBatch)."""
        return self._query_batch("count", n_streams, overlapping)

    def is_match_stream(self, patterns=None) -> TokenStream:
        return self._query_stream("is_match", False, patterns)

    def find_first_stream(self, patterns=None) -> TokenStream:
        return self._query_stream("find_first", False, patterns)

    def count_matches_stream(self, overlapping: bool = False) -> TokenStream:
        self._ac.check_overlapping(overlapping)
        return self._query_stream("count", overlapping)

    def match_mask_stream_batch(self, n_streams: int, overlapping: bool = False, pattern_sets=None, set_index=None) -> TokenStreamBatch:
        """``feed_device(tokens, offsets, last=None)`` -> (flags, flag_offsets, flag_starts), a flag per token for each
        stream's tokens that no later ids can change: all but the last k - 1 fed, k the longest pattern in tokens (see
        MaskStreamBatch).  Masking banned sequences as a model emits them.  pattern_sets= / set_index= (n_streams,)."""
        _token_stream_limits(self._ac, n_streams)
        return TokenStreamBatch(_mask_stream_batch(self._ac, n_streams, overlapping, pattern_sets, set_index, _capi.ACB_TOKEN_BYTES), _same)

    def match_spans_stream(self, overlapping: bool = False, patterns=None) -> "TokenMaskStream":
        """One match-mask stream fed host chunks of ids: ``feed(chunk)`` -> the runs (start, end) of covered tokens this
        feed released, ``finish()`` -> the rest (see MaskStream)."""
        _token_stream_limits(self._ac, 1)
        return TokenMaskStream(_mask_stream(self._ac, overlapping, False, patterns, _capi.ACB_TOKEN_BYTES), _same)


def _token_tuples_of_rows(rows):
    return [(p, s // _capi.ACB_TOKEN_BYTES, e // _capi.ACB_TOKEN_BYTES) for p, s, e in rows]
