"""Vocabulary masks without a DFA walk: which next ids complete a pattern, from the contract's decomposition alone.

Id t completes an admitted pattern p after the history's bytes T (those after its last break) in one of two ways:
p occurs inside vocab[t]; or, for some 1 <= k < len(p), T ends with p[:k] and vocab[t] starts with p[k:].  The first
part does not depend on T: one Standard overlapping oracle search over all entries joined, keeping each match that lies
inside one entry (an overlapping search reports every occurrence, so no separator is needed).  The second is a lookup
of the last 1 .. max_pattern_len - 1 bytes of T among the patterns' proper prefixes, each remainder p[k:] becoming an
id range of the entries sorted by their bytes.  Nothing here reads the vocabulary image (trans, colmap, depth, lvl2,
tail_hit), so it checks the kernels and the interpreter in tests/vocab_model.py alike, at a million entries."""
from bisect import bisect_left

import numpy as np
import torch

from oracle import Oracle


def tail_bytes(vocab, history):
    """T: the bytes of the history after its last break (an id outside [0, n_vocab))."""
    h = [int(x) for x in history]
    n = len(vocab)
    i = len(h)
    while i and 0 <= h[i - 1] < n:
        i -= 1
    return b"".join(vocab[x] for x in h[i:])


def row_history(flat, offsets, i):
    """Row i's ids under the kernels' offset rule: offsets[i], offsets[i + 1] clamped to [0, len(flat)], b < a empty."""
    a, b = (min(max(int(x), 0), len(flat)) for x in (offsets[i], offsets[i + 1]))
    return list(flat[a:b]) if b >= a else []


def _successor(r: bytes):
    """The least byte string above every string that starts with r, or None when there is none (r is all 0xff)."""
    r = r.rstrip(b"\xff")
    return r[:-1] + bytes([r[-1] + 1]) if r else None


class VocabReference:
    def __init__(self, patterns, vocab):
        self.pats = [bytes(p) for p in patterns]
        self.vocab = [bytes(v) for v in vocab]
        n = self.n_vocab = len(self.vocab)
        self.K = max((len(p) for p in self.pats), default=0)
        offs = np.zeros(n + 1, dtype=np.int64)
        if n:
            np.cumsum(np.fromiter((len(v) for v in self.vocab), dtype=np.int64, count=n), out=offs[1:])
        self._hit_id = self._hit_pid = np.zeros(0, dtype=np.int64)
        if self.pats and offs[-1]:
            blob = np.frombuffer(b"".join(self.vocab), dtype=np.uint8)
            _, _, rec = Oracle(self.pats, "Standard").scan_batch(blob, np.array([0, offs[-1]], dtype=np.int64), overlapping=True)
            pid, s, e = (rec[:, c].astype(np.int64) for c in (1, 2, 3))
            t = np.searchsorted(offs, s, side="right") - 1   # the non-empty entry the match starts in
            inside = e <= offs[t + 1]
            self._hit_id, self._hit_pid = t[inside], pid[inside]
        self.order = np.array(sorted(range(n), key=self.vocab.__getitem__), dtype=np.int64)
        self.sorted = [self.vocab[t] for t in self.order]
        self.heads = {}   # p[:k] -> [(pid, p[k:])] for 1 <= k < len(p)
        for pid, p in enumerate(self.pats):
            for k in range(1, len(p)):
                self.heads.setdefault(p[:k], []).append((pid, p[k:]))
        self._contains = {}

    def contains(self, admitted=None):
        """The ids that hold an occurrence of an admitted pattern (sorted, distinct)."""
        key = None if admitted is None else frozenset(admitted)
        got = self._contains.get(key)
        if got is None:
            ids = self._hit_id if key is None else self._hit_id[np.isin(self._hit_pid, np.fromiter(key, dtype=np.int64))]
            got = self._contains[key] = np.unique(ids)
        return got

    def starting_with(self, r: bytes):
        """The ids whose bytes start with r."""
        lo = bisect_left(self.sorted, r)
        nxt = _successor(r)
        hi = self.n_vocab if nxt is None else bisect_left(self.sorted, nxt, lo)
        return self.order[lo:hi]

    def banned_tail(self, T: bytes, admitted=None, V=None):
        """The sorted ids below min(V, n_vocab) that complete an admitted pattern after the bytes T."""
        parts = [self.contains(admitted)]
        for k in range(1, min(len(T), self.K - 1) + 1):
            for pid, rest in self.heads.get(T[len(T) - k:], ()):
                if admitted is None or pid in admitted:
                    parts.append(self.starting_with(rest))
        out = np.unique(np.concatenate(parts))
        lim = self.n_vocab if V is None else min(V, self.n_vocab)
        return out[out < lim]

    def __call__(self, history, admitted=None, V=None):
        """As BruteModel: the sorted list of ids that complete an admitted pattern after `history`."""
        return self.banned_tail(tail_bytes(self.vocab, history), admitted, V).tolist()

    def table(self, histories, V, admitted=None, device="cuda"):
        """(len(histories), V) bool tensor on `device`: row d bans what history d bans.  `admitted`: None, or one set
        (or None) per history."""
        out = torch.zeros(len(histories), V, dtype=torch.bool, device=device)
        for d, h in enumerate(histories):
            ids = self.banned_tail(tail_bytes(self.vocab, h), None if admitted is None else admitted[d], V)
            if ids.size:
                out[d, torch.from_numpy(ids).to(device)] = True
        return out


def expected_logits(before, ban, value):
    """`before` with value -- rounded from float32 to the logits dtype on the device, as torch rounds it -- where `ban`
    holds, and bit-identical elsewhere."""
    fill = torch.tensor([value], dtype=torch.float32, device=before.device).to(before.dtype)
    return torch.where(ban, fill, before)


def bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32)
