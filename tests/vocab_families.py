"""Seeded (patterns, vocabulary, histories) families aimed at the vocabulary kernels' geometry (csrc/vocab.cuh): the
state kernel's 32-id history pieces, the mask kernel's walk branches and the DFA shapes of tests/table_shapes.py.
Shared by the CPU cross-check of the reference (tests/test_vocab_reference_cpu.py) and the GPU tests
(tests/test_gpu_vocab_geometry.py)."""
import numpy as np

from . import table_shapes as ts

PIECE_LENS = (33, 64, 65, 100, 1000)   # need = 32 .. 999 bytes: 1 to 32 pieces of one-byte ids
ALPHA = b"abcd"


def _rand(rng, alpha, k):
    return np.frombuffer(alpha, dtype=np.uint8)[rng.integers(0, len(alpha), k)].tobytes()


def _split(rng, text, k):
    """text cut into k consecutive pieces, some of them empty."""
    cuts = sorted(int(x) for x in rng.integers(0, len(text) + 1, max(k - 1, 0)))
    edges = [0] + cuts + [len(text)]
    return [text[edges[i]:edges[i + 1]] for i in range(k)]


class Family:
    """patterns, vocab (list of bytes) and histories (lists of ids), built from histories written as byte segments:
    every distinct segment becomes an entry after the `base` entries; None in a history is a break."""

    def __init__(self, name, patterns, base, seg_histories):
        self.name, self.patterns = name, [bytes(p) for p in patterns]
        self.vocab = list(base)
        index = {}
        for t, v in enumerate(self.vocab):
            index.setdefault(v, t)
        for h in seg_histories:
            for s in h:
                if s is not None and s not in index:
                    index[s] = len(self.vocab)
                    self.vocab.append(s)
        n = len(self.vocab)
        self.histories = [[n + 3 if s is None else index[s] for s in h] for h in seg_histories]
        self.need = max(max((len(p) for p in self.patterns), default=0) - 1, 0)


def read_stop(vocab, history, need):
    """The id index k (counted back from the row's end, 0 = the last id) at which vocab_state_kernel's backwards scan
    stops: `need` bytes reached, a break, or the row start (k = the row's length).  None when need is 0."""
    if not need:
        return None
    cum = 0
    for k in range(len(history)):
        t = int(history[len(history) - 1 - k])
        if not 0 <= t < len(vocab):
            return k
        cum += len(vocab[t])
        if cum >= need:
            return k
    return len(history)


def pieces(L, seed=0):
    """A pattern P of L bytes over ALPHA (and P[5:8]), over one-byte ids, empty ids and pieces of P.  Histories end in
    P[:need] (so its last byte completes P) with the scan stopping by reach at lane 0 or 31 of pieces 0-3, with
    cum == need (skip 0) and with a long id straddling the cut (also where the history holds all of P); others stop at a break at a piece boundary or at the
    row start after 32, 33 and 64 ids; junk, empty ids and breaks before the stop must not matter."""
    rng = np.random.default_rng(100 + L + seed)
    P = _rand(rng, ALPHA, L)
    need = L - 1
    base = [bytes([b]) for b in ALPHA] + [b""]
    hists = []

    def junk():
        out = [bytes([b]) for b in _rand(rng, ALPHA, int(rng.integers(0, 40)))]
        for _ in range(int(rng.integers(0, 3))):
            out.insert(int(rng.integers(0, len(out) + 1)), [None, b""][int(rng.integers(0, 2))])
        return out

    for k in (0, 31, 32, 63, 64, 95, 96, int(rng.integers(97, 1100))):
        for skip in (0, 3):
            lk = skip + 1 + int(rng.integers(0, min(6, need) + 1))   # the stopping id's length
            text = _rand(rng, ALPHA, skip) + P[:need]
            s = need + skip - lk                                     # bytes of the k ids after it
            if s < 0 or (k == 0 and s):
                continue
            hists.append(junk() + [text[:lk]] + _split(rng, text[lk:], k))
    for skip in (1, 3):   # all of P, the stopping id straddling the cut: a walk over more bytes would end in P's state
        text = _rand(rng, ALPHA, skip) + P
        hists.append(junk() + [text[:skip + 2]] + _split(rng, text[skip + 2:], int(rng.integers(1, 40))))
    # full one-byte spelling, with and without empty ids between the bytes
    hists.append(junk() + [bytes([b]) for b in P[:need]])
    spelled = []
    for b in P[:need]:
        spelled += [bytes([b])] + [b""] * int(rng.integers(0, 3))
    hists.append(spelled)
    # a break at k = 31, 32, 64, and the row start after 32, 33, 64 ids: fewer than `need` bytes after either
    for k in (31, 32, 64):
        m = min(need - 1, int(rng.integers(k // 2, k + 40)))
        hists.append(junk() + [None] + _split(rng, P[:m], k))
    for k in (32, 33, 64):
        m = min(need - 1, int(rng.integers(k // 2, k + 40)))
        hists.append(_split(rng, P[:m], k))
    for _ in range(6):   # random tokenizations of a random prefix of P, after junk
        m = int(rng.integers(0, L))
        hists.append(junk() + _split(rng, P[:m], int(rng.integers(0, 2 * m + 2))))
    return Family(f"pieces-{L}", [P, P[5:8]], base, hists)


def dam_then_empties():
    """b"dam", then 1000 empty ids: the scan reads 32 pieces without a byte before it reaches "dam"; "n" completes."""
    base = [b"d", b"am", b"dam", b"", b"n", b"x", b"amn"]
    hists = [[b"dam"] + [b""] * 1000, [b"d", b"am"] + [b""] * 999, [b"x"] + [b""] * 1000, [b""] * 1001]
    return Family("dam-empties", [b"damn"], base, hists)


def one_byte():
    """Only one-byte patterns: need = 0 and no state of depth 2 (lvl2 == n_states)."""
    base = [b"a", b"b", b"\x00", b"ba", b"", b"bbb", b"\xff", b"xyz"]
    hists = [[], [b"a"], [None], [b"bbb", b"b"]]
    return Family("one-byte", [b"a", b"\x00", b"a", b"\xff"], base, hists)


def deep_state(seed=0):
    """A 200-byte pattern: a row state of depth 100+ and candidates up to 150 bytes that stay deep, diverge late or
    complete it."""
    rng = np.random.default_rng(300 + seed)
    P = _rand(rng, b"ab", 200)
    pats = [P, b"ba" * 3, b"abb"]
    base = [b"a", b"b", b""]
    for cut in (120, 150, 199):
        for k in (1, 20, 79, 80, 81, 150):
            c = P[cut:cut + k]
            base.append(c)
            if c:
                base.append(c[:-1] + (b"a" if c[-1:] == b"b" else b"b"))
    base.append(P[50:200])
    hists = [[bytes([b]) for b in P[:cut]] for cut in (120, 150, 199, 101)]
    hists += [[P[:60], P[60:150]], [b"b" * 3, P[:120]], [None, P[:120]]]
    return Family("deep-state", pats, base, hists)


def filtered_tails():
    """Candidates whose tail_hit lies past the depth stop: with no admitted hit at all, and with the only admitted hit
    at the tail_hit byte; nested and duplicate patterns whose sets admit only a suffix pid."""
    pats = [b"xy", b"zw", b"abc", b"bc", b"bc", b"c"]
    base = [b"qqxyqqzw", b"qqxyqq", b"qqzw", b"zw", b"xy", b"q", b"x", b"y", b"z", b"w", b"", b"abc", b"bc", b"c", b"a",
            b"b", b"qabcq", b"qqqqqqqqqqxy", b"wqqqqqqqqqqqqqqzw"]
    hists = [[], [b"x"], [b"z"], [b"a"], [b"a", b"b"], [b"b"], [b"q"], [None]]
    return Family("filtered-tails", pats, base, hists)


def shadowed():
    """[ab, abcd]: under LeftmostFirst abcd is shadowed by ab; a set admitting only pid 1 must still ban its
    completions (the image's Standard DFA)."""
    base = [b"a", b"b", b"c", b"d", b"ab", b"cd", b"abcd", b"bcd", b"d!", b""]
    hists = [[], [b"a"], [b"ab"], [b"a", b"b", b"c"], [b"ab", b"c"], [b"a", b"bcd"]]
    return Family("shadowed", [b"ab", b"abcd"], base, hists)


WALKS = [one_byte, deep_state, filtered_tails, shadowed, dam_then_empties]


def shape_family(case, seed=0, n_hist=24):
    """A tests/table_shapes case as a vocabulary: single bytes of its alphabet, bytes outside it and Case.outside bytes,
    prefixes, suffixes and pieces of its patterns; histories of random ids and of pattern prefixes."""
    rng = np.random.default_rng(500 + seed + ts.CASE_IDS.index(case.name))
    al = bytes(case.alphabet)
    outside = bytes(b for b in range(256) if b not in set(al))
    base = [bytes([b]) for b in al[:64]] + [bytes([b]) for b in outside[::7]] + [bytes([b]) for b in case.outside[:16]] + [b""]
    for p in case.pats[:80]:
        k = int(rng.integers(1, len(p) + 1))
        base += [p[:k], p[k:], p[max(k - 2, 0):k + 2]]
    if case.outside:   # decoys: a pattern starting with the highest byte, with an outside byte in its place
        top = max(case.alphabet)
        base += [bytes([case.outside[i % len(case.outside)]]) + p[1:] for i, p in enumerate(case.pats) if p[0] == top][:8]
    base = [b for b in dict.fromkeys(base)]
    hists = [[]]
    for i in range(n_hist):
        p = case.pats[int(rng.integers(0, len(case.pats)))]
        h = [bytes(base[int(x)]) for x in rng.integers(0, len(base), int(rng.integers(0, 6)))]
        if i % 2:
            k = int(rng.integers(1, len(p))) if len(p) > 1 else 1
            h += [p[:k]]
        hists.append(h)
    return Family(f"shape-{case.name}", case.pats, base, hists)


def stride_vocab(rng, n_vocab, alpha=b"abcdefgh"):
    """n_vocab seeded entries of 0-4 bytes over `alpha` (the single bytes first) and patterns that ban ids up to the
    last one: substrings of the vocabulary's own entries and pairs of them."""
    vocab = [bytes([b]) for b in alpha]
    while len(vocab) < n_vocab:
        vocab.append(_rand(rng, alpha, int(rng.integers(0, 5))))
    vocab = vocab[:n_vocab]
    pats = [vocab[-1] or b"a", b"abc", b"ha", b"gfe", b"dddd", b"bahg", b"cg"]
    pats += [vocab[int(i)] + vocab[int(j)] for i, j in rng.integers(8, n_vocab, (12, 2)) if vocab[int(i)] + vocab[int(j)]]
    return [p for p in pats if p], vocab


def all_strings(alpha: bytes, max_len, seed):
    """Every 1- to max_len-byte string over alpha, in a seeded shuffle."""
    out = [bytes([b]) for b in alpha]
    layer = out
    for _ in range(max_len - 1):
        layer = [s + bytes([b]) for s in layer for b in alpha]
        out += layer
    rng = np.random.default_rng(seed)
    return [out[int(i)] for i in rng.permutation(len(out))]
