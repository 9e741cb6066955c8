"""Vocabulary masks without a GPU: two independent statements of which next ids complete a string pattern.

1. ``brute_completing``: the contract itself over the oracle.  T is the history's bytes after its last break (an id
   outside [0, n_vocab)); id t completes a pattern when a Standard overlapping search of T + vocab[t] has a match of an
   admitted pattern ending past len(T).  Filtering the overlapping list by pid afterwards is exact.
2. ``VocabImage``: an interpreter of acb_vocab_write's bytes that does what the kernels do (csrc/vocab.cuh): the
   backwards tail decode, the forward walk of the row's state, and per candidate the walk with the depth / tail_hit
   early stop, the filtered path included."""
import ctypes as C
import struct

import numpy as np

from ahocorasick_rs_b200 import _capi
from oracle import Oracle

MATCH = 0x80000000
MASK = 0x7FFFFFFF
ROOT = 1


def decoded_tail(vocab, history):
    """T: the bytes of the history after its last break."""
    out = b""
    for c in history:
        c = int(c)
        out = out + vocab[c] if 0 <= c < len(vocab) else b""
    return out


class BruteModel:
    """brute_completing with the oracle built once (all patterns, kind Standard), for many histories."""

    def __init__(self, patterns, vocab):
        self.vocab = [bytes(v) for v in vocab]
        self.orc = Oracle([bytes(p) for p in patterns], "Standard") if patterns else None

    def __call__(self, history, admitted=None, V=None):
        if self.orc is None:
            return []
        T = decoded_tail(self.vocab, history)
        n = len(self.vocab) if V is None else min(V, len(self.vocab))
        out = []
        for t in range(n):
            if any(e > len(T) and (admitted is None or p in admitted) for p, _, e in self.orc.find(T + self.vocab[t], overlapping=True)):
                out.append(t)
        return out


def brute_completing(patterns, vocab, history, admitted=None, V=None):
    return BruteModel(patterns, vocab)(history, admitted, V)


def build_automaton(patterns, kind=0):
    L = _capi.lib()
    offs = np.zeros(len(patterns) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in patterns], out=offs[1:])
    blob = np.frombuffer(b"".join(bytes(p) for p in patterns) or b"\0", dtype=np.uint8)
    h = C.c_void_p()
    rc = L.acb_build(blob.ctypes.data, offs.ctypes.data, len(patterns), kind, -1, C.byref(h))
    assert rc == _capi.ACB_OK, _capi.last_error()
    return L, h


def pack_vocab(vocab):
    offs = np.zeros(len(vocab) + 1, dtype=np.uint64)
    np.cumsum([len(v) for v in vocab], out=offs[1:])
    blob = np.frombuffer(b"".join(bytes(v) for v in vocab) or b"\0", dtype=np.uint8)
    return blob, offs


def image_bytes(patterns, vocab, kind=0):
    """The vocabulary image, as acb_vocab_write gives it."""
    L, h = build_automaton(patterns, kind)
    try:
        blob, offs = pack_vocab(vocab)
        n = C.c_uint64(0)
        assert L.acb_vocab_build(h, blob.ctypes.data, offs.ctypes.data, len(vocab), C.byref(n)) == _capi.ACB_OK, _capi.last_error()
        buf = np.zeros(n.value, dtype=np.uint8)
        assert L.acb_vocab_write(h, blob.ctypes.data, offs.ctypes.data, len(vocab), buf.ctypes.data, n.value) == _capi.ACB_OK
        return buf.tobytes()
    finally:
        L.acb_free(h)


class VocabImage:
    """Reads a vocabulary image: header (magic, n_vocab, n_states, n_cols, max_pat_len, lvl2, n_tail_hits, pad, then the
    u64 extra DFA bytes and the offsets of the DFA, its transitions, colmap, match_off and match_pid, depth, records,
    tail_hit and the entry bytes, and the total size)."""

    def __init__(self, buf: bytes):
        (self.magic, self.n_vocab, self.n_states, self.n_cols, self.max_pat_len, self.lvl2, self.n_tail_hits,
         _) = struct.unpack_from("<8I", buf, 0)
        (self.extra, self.off_dfa, off_trans, off_colmap, off_moff, off_mpid, off_depth, off_recs, off_tail, off_bytes,
         self.total) = struct.unpack_from("<11Q", buf, 32)
        assert self.total == len(buf)
        self.trans = np.frombuffer(buf, dtype=np.uint32, count=self.n_states * self.n_cols, offset=off_trans).reshape(-1, self.n_cols)
        self.colmap = np.frombuffer(buf, dtype=np.uint8, count=256, offset=off_colmap)
        self.match_off = np.frombuffer(buf, dtype=np.uint32, count=self.n_states + 1, offset=off_moff)
        self.match_pid = np.frombuffer(buf, dtype=np.uint32, count=int(self.match_off[-1]), offset=off_mpid)
        self.depth = np.frombuffer(buf, dtype=np.uint32, count=self.n_states, offset=off_depth)
        self.recs = np.frombuffer(buf, dtype=np.uint32, count=2 * self.n_vocab, offset=off_recs).reshape(-1, 2)
        self.tail = np.frombuffer(buf, dtype=np.int32, count=self.n_vocab, offset=off_tail)
        n_bytes = int(self.recs[-1, 0] + self.recs[-1, 1]) if self.n_vocab else 0
        self.bytes = np.frombuffer(buf, dtype=np.uint8, count=n_bytes, offset=off_bytes)
        self.need = max(self.max_pat_len - 1, 0)

    def entry(self, t):
        o, n = (int(x) for x in self.recs[t])
        return self.bytes[o:o + n]

    def step(self, s, byte):
        return int(self.trans[s, self.colmap[byte]])

    def state(self, history):
        """vocab_state_kernel: back over the ids until `need` bytes, a break or the row start, then forward from the root."""
        hist = [int(x) for x in history]
        have, start, skip = 0, len(hist), 0
        if self.need:
            for i in range(len(hist) - 1, -2, -1):
                if i < 0 or not 0 <= hist[i] < self.n_vocab:
                    start, skip = i + 1, 0
                    break
                ln = int(self.recs[hist[i], 1])
                if have + ln >= self.need:
                    start, skip = i, have + ln - self.need
                    break
                have += ln
        s = ROOT
        for i in range(start, len(hist)):
            for b in self.entry(hist[i])[skip if i == start else 0:]:
                s = self.step(s, b) & MASK
        return s

    def hit(self, e, admitted):
        if not e & MATCH:
            return False
        if admitted is None:
            return True
        s = e & MASK
        return any(int(p) in admitted for p in self.match_pid[self.match_off[s]:self.match_off[s + 1]])

    def banned(self, s, t, admitted=None):
        """vocab_banned: the walk from the row's state with the depth / tail_hit early stop."""
        tok = self.entry(t)
        if len(tok) == 0:
            return False
        tail = int(self.tail[t])
        e = self.step(s, tok[0])
        if self.hit(e, admitted):
            return True
        s, j = e & MASK, 0
        if s >= self.lvl2:
            while True:
                j += 1
                if j == len(tok):
                    return False
                e = self.step(s, tok[j])
                if self.hit(e, admitted):
                    return True
                s = e & MASK
                if self.depth[s] <= j + 1:
                    break
        if tail <= j:
            return False
        if admitted is None:
            return True
        while j + 1 <= tail:
            j += 1
            e = self.step(s, tok[j])
            if self.hit(e, admitted):
                return True
            s = e & MASK
        return False

    def completing(self, history, admitted=None, V=None):
        s = self.state(history)
        n = self.n_vocab if V is None else min(V, self.n_vocab)
        return [t for t in range(n) if self.banned(s, t, admitted)]

    def first_byte_ids(self, history):
        """How many non-empty ids the walk from the row's state decides on their first byte."""
        s = self.state(history)
        return sum(1 for t in range(self.n_vocab) if len(self.entry(t)) and
                   ((self.step(s, self.entry(t)[0]) & MATCH) or (self.step(s, self.entry(t)[0]) & MASK) < self.lvl2))


def direct_depth(trans):
    """The length of the string each state spells, as its distance from the root over the dense table (BFS)."""
    n = trans.shape[0]
    depth = np.full(n, -1, dtype=np.int64)
    depth[ROOT] = 0
    frontier = [ROOT]
    d = 0
    while frontier:
        d += 1
        nxt = []
        for s in frontier:
            for t in set(int(x) & MASK for x in trans[s]):
                if depth[t] < 0:
                    depth[t] = d
                    nxt.append(t)
        frontier = nxt
    return depth


def direct_tail_hit(patterns, vocab):
    """tail_hit of every entry from the oracle: the last end - 1 of its own overlapping matches, -1 for none."""
    if not patterns:
        return [-1] * len(vocab)
    orc = Oracle([bytes(p) for p in patterns], "Standard")
    return [max((e - 1 for _, _, e in orc.find(bytes(v), overlapping=True)), default=-1) for v in vocab]
