"""Completing tokens without a GPU: the brute-force statement of the contract, and an interpreter of the completions image
(csrc/completions.h) that walks it as the kernel does (csrc/completions.cuh), including the first-occurrence rule the
count and emit modes report by.

Id t COMPLETES a pattern for history C when some admitted p is a suffix of C + [t]: p[:-1] is a suffix of C and
p[-1] == t.  Only the suffixes of C up to K - 1 ids long matter (K = the longest pattern)."""
import ctypes as C
import struct

import numpy as np

from ahocorasick_rs_b200 import _capi

LIMIT = _capi.ACB_TOKEN_ID_LIMIT
# the edge ids of the token format (tests/test_gpu_tokens.py): each byte at 0 and 127, the 7-bit carries, the largest id
ALPHA = [0, 1, 127, 128, 5, 5 + (1 << 7), 5 + (1 << 14), 1 << 14, (1 << 14) + 1, 1 + (1 << 7), (1 << 21) - 1]


def model_completing(patterns, history, admitted=None):
    """The statement: map tuple(p[:-1]) to the set of p[-1] over admitted patterns, then look up every suffix of the
    history up to K - 1 ids.  -> sorted list of distinct ids."""
    return CompletionModel(patterns, admitted)(history)


class CompletionModel:
    """model_completing with its table built once, for many histories."""

    def __init__(self, patterns, admitted=None):
        self.table = {}
        self.K = 0
        for pid, p in enumerate(patterns):
            self.K = max(self.K, len(p))
            if admitted is None or pid in admitted:
                self.table.setdefault(tuple(int(x) for x in p[:-1]), set()).add(int(p[-1]))

    def __call__(self, history):
        hist = [int(x) for x in history]
        out = set()
        for d in range(0, min(len(hist), self.K - 1) + 1) if self.K else ():
            out |= self.table.get(tuple(hist[len(hist) - d:]), set())
        return sorted(out)


def encode(ids):
    """The token format (include/acb200.h) stated again: 0x80 | t >> 14, (t >> 7) & 0x7f, t & 0x7f per id."""
    t = np.asarray(ids, dtype=np.int64).reshape(-1)
    out = np.empty((len(t), 3), dtype=np.uint8)
    out[:, 0] = 0x80 | (t >> 14)
    out[:, 1] = (t >> 7) & 0x7F
    out[:, 2] = t & 0x7F
    return out.tobytes()


def build_automaton(pattern_bytes, kind=0):
    """acb_build on raw byte patterns -> (lib, handle); the caller frees the handle."""
    L = _capi.lib()
    offs = np.zeros(len(pattern_bytes) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pattern_bytes], out=offs[1:])
    blob = np.frombuffer(b"".join(pattern_bytes) or b"\0", dtype=np.uint8)
    h = C.c_void_p()
    rc = L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pattern_bytes), kind, -1, C.byref(h))
    assert rc == _capi.ACB_OK, _capi.last_error()
    return L, h


def image_bytes(patterns, kind=0):
    """The completions image of token-id patterns, as acb_completions_write gives it."""
    L, h = build_automaton([encode(p) for p in patterns], kind)
    try:
        n = C.c_uint64(0)
        assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_OK, _capi.last_error()
        buf = np.zeros(n.value, dtype=np.uint8)
        assert L.acb_completions_write(h, buf.ctypes.data, n.value) == _capi.ACB_OK
        return buf.tobytes()
    finally:
        L.acb_free(h)


NONE = 0xFFFFFFFF


class ComplImage:
    """Reads a completions image: header (magic, n_nodes, n_entries, depth, max_last, 3 x pad, then the u64 offsets of
    the nodes, the child tokens and the entries, and the total size), nodes of 8 u32 (first_kid, n_kids, first_entry,
    n_entries, elink, 3 x pad), u32 child tokens, entries of 2 u32 (token, pid)."""

    def __init__(self, buf: bytes):
        self.magic, self.n_nodes, self.n_entries, self.depth, self.max_last = struct.unpack_from("<5I", buf, 0)
        off_nodes, off_kid, off_entries, self.total = struct.unpack_from("<4Q", buf, 32)
        assert self.total == len(buf)
        self.nodes = np.frombuffer(buf, dtype=np.uint32, count=8 * self.n_nodes, offset=off_nodes).reshape(-1, 8)
        self.kid_tok = np.frombuffer(buf, dtype=np.uint32, count=self.n_nodes, offset=off_kid)
        self.entries = np.frombuffer(buf, dtype=np.uint32, count=2 * self.n_entries, offset=off_entries).reshape(-1, 2)

    def path(self, history):
        """The nodes the walk visits, root first: one per suffix of the history (up to `depth` ids) that is some p[:-1]."""
        hist = [int(x) for x in history]
        m = min(len(hist), self.depth)
        v, out = 0, [0]
        for d in range(m):
            t = hist[len(hist) - 1 - d]
            if not 0 <= t < LIMIT:
                break
            fk, nk = int(self.nodes[v, 0]), int(self.nodes[v, 1])
            kids = self.kid_tok[fk:fk + nk]
            j = int(np.searchsorted(kids, t))
            if j == nk or kids[j] != t:
                break
            v = fk + j
            out.append(v)
        return out

    def node_entries(self, v):
        fe, ne = int(self.nodes[v, 2]), int(self.nodes[v, 3])
        return [(int(t), int(p)) for t, p in self.entries[fe:fe + ne]]

    def completing(self, history, admitted=None):
        """What the mask mode writes: every admitted entry's token along the path."""
        return sorted({t for v in self.path(history) for t, p in self.node_entries(v) if admitted is None or p in admitted})

    def emitted(self, history, admitted=None):
        """What the emit mode writes, in its order: per node (root first), per entry, the entries that are their token's
        first admitted occurrence -- none earlier in the node, none at an ancestor reached through elink."""
        ok = (lambda p: True) if admitted is None else (lambda p: p in admitted)
        out = []
        for v in self.path(history):
            ents = self.node_entries(v)
            for i, (t, p) in enumerate(ents):
                if not ok(p) or any(t2 == t and ok(p2) for t2, p2 in ents[:i]):
                    continue
                u, seen = int(self.nodes[v, 4]), False
                while u != NONE:
                    seen |= any(t2 == t and ok(p2) for t2, p2 in self.node_entries(u))
                    u = int(self.nodes[u, 4])
                if not seen:
                    out.append(t)
        return out

    def check_structure(self, patterns):
        """The layout's invariants: breadth-first children, sorted child tokens and entries, elink = the nearest proper
        ancestor with entries, the header's depth and max_last, and every pattern as exactly one entry."""
        assert self.magic == 0x31434341
        parent = [NONE] * self.n_nodes
        for v in range(self.n_nodes):
            fk, nk = int(self.nodes[v, 0]), int(self.nodes[v, 1])
            if nk:
                assert fk > v and fk + nk <= self.n_nodes
                assert np.all(np.diff(self.kid_tok[fk:fk + nk].astype(np.int64)) > 0)
            for c in range(fk, fk + nk):
                parent[c] = v
            ents = self.node_entries(v)
            assert ents == sorted(ents)
        assert all(parent[v] != NONE for v in range(1, self.n_nodes))
        for v in range(self.n_nodes):
            u = parent[v]
            while u != NONE and self.nodes[u, 3] == 0:
                u = parent[u]
            assert int(self.nodes[v, 4]) == u
        assert self.n_entries == len(patterns)
        assert self.depth == max((len(p) - 1 for p in patterns), default=0)
        assert self.max_last == max((int(p[-1]) for p in patterns), default=0)
        got = {}
        for v in range(self.n_nodes):
            for t, p in self.node_entries(v):
                got[p] = (v, t)
        assert sorted(got) == list(range(len(patterns)))
        for pid, p in enumerate(patterns):   # the entry's node spells p[:-1]: each node prepends its token to its parent's
            v, t = got[pid]
            assert t == int(p[-1])
            spelled = []
            while v != 0:
                spelled.append(int(self.kid_tok[v]))
                v = parent[v]
            assert spelled == [int(x) for x in p[:-1]]


def random_patterns(rng, n, max_len, alphabet):
    """Seeded pattern lists with one-token patterns, duplicates, nested patterns, shared prefixes and many patterns
    that share a last token."""
    pats = [[int(x) for x in rng.choice(alphabet, int(rng.integers(1, max_len + 1)))] for _ in range(n)]
    if pats:
        pats.append(list(pats[0]))                                  # a duplicate
        pats.append(pats[-1][-1:])                                  # a one-token suffix of it
        base = [int(x) for x in rng.choice(alphabet, max_len)]
        pats += [base[i:] for i in range(len(base))]                # nested: every suffix
        pats += [base[:i] for i in range(1, len(base) + 1)]         # shared prefixes
        last = int(rng.choice(alphabet))
        pats += [[int(x) for x in rng.choice(alphabet, int(rng.integers(0, max_len)))] + [last] for _ in range(8)]
    return pats
