"""GPU tests of the match-mask streams (-m gpu): MaskStreamBatch.feed_device on the three classes and the host forms.
After every feed, each stream's released flags equal match_mask_device of its whole concatenation at those positions,
and flag_offsets / flag_starts equal the release rule R = max(0, F - (max_pattern_len - 1)) (R = F on `last`), in
bytes, or in tokens at their first byte.  Ragged chunks over many streams (empty ones, `last` on a subset mid-run, slots
reused), a generation loop of one token per stream per feed, pattern sets (an index outside [0, n_sets) gives all
False), patterns of 300-3000 bytes, max_pattern_len 1, non-default sieve geometries, the host forms against
match_spans, two threads."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, dev  # noqa: E402

TUNINGS = {"default": (0, 0, 0, 0, 0), "small-tasks": (5, 0, 512, 0, 0), "ring-1": (5, 0, 512, 0, 1)}
TOKEN_DTYPES = [torch.uint16, torch.int32, torch.int64]


class tuned:
    def __init__(self, name):
        self.t = TUNINGS[name]

    def __enter__(self):
        _capi.set_tuning(*self.t)

    def __exit__(self, *exc):
        _capi.set_tuning()


class Units:
    """How a class's sequences go to the device: bytes (str and bytes classes) or token ids of one dtype."""

    def __init__(self, ac, tokens_dtype=None):
        self.ac, self.dtype = ac, tokens_dtype
        self.unit = _capi.ACB_TOKEN_BYTES if tokens_dtype is not None else 1
        self.halo = ac._ac.max_pattern_len - 1

    def to_dev(self, arr):
        if self.dtype is None:
            return dev(np.asarray(arr, dtype=np.uint8))
        return torch.from_numpy(np.asarray(arr, dtype=np.int64)).cuda().to(self.dtype)

    def reference(self, seqs, pattern_sets=None, set_index=None):
        """match_mask_device of each sequence whole, one batch -> a bool numpy mask per sequence (per unit)."""
        offs = np.zeros(len(seqs) + 1, dtype=np.int64)
        np.cumsum([len(s) for s in seqs], out=offs[1:])
        data = np.concatenate([np.asarray(s, dtype=np.int64) for s in seqs] + [np.zeros(0, dtype=np.int64)])
        m = self.ac.match_mask_device(self.to_dev(data), dev(offs), self.overlapping, pattern_sets=pattern_sets, set_index=set_index)
        m = m.cpu().numpy()
        return [m[offs[i]:offs[i + 1]] for i in range(len(seqs))]


def run_streams(u, batch, queues, rng, step_max, refs, one_step=False, last_p=0.7):
    """Feeds the queues (per slot, a list of sequences; a slot starts its next sequence after `last`) in random steps and
    checks every feed against the reference masks `refs` (same nesting).  -> the number of sequences finished."""
    n = len(queues)
    pos, cur, fed_bytes, done = [0] * n, [0] * n, [0] * n, 0
    got = [[] for _ in range(n)]
    while any(c < len(q) for c, q in zip(cur, queues)):
        chunks, last = [], np.zeros(n, dtype=bool)
        for i in range(n):
            if cur[i] >= len(queues[i]):
                chunks.append(np.zeros(0, dtype=np.int64))
                continue
            seq = queues[i][cur[i]]
            k = 1 if one_step else (0 if rng.random() < 0.15 else int(rng.integers(1, step_max + 1)))
            chunks.append(np.asarray(seq[pos[i]:pos[i] + k], dtype=np.int64))
            pos[i] = min(len(seq), pos[i] + k)
            last[i] = pos[i] == len(seq) and rng.random() < last_p
        offs = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([len(c) for c in chunks], out=offs[1:])
        flags, fo, fs = batch.feed_device(u.to_dev(np.concatenate(chunks)), dev(offs), dev(last) if last.any() else None)
        flags, fo, fs = flags.cpu().numpy(), fo.cpu().numpy(), fs.cpu().numpy()
        assert flags.dtype == bool and fo[0] == 0 and fo[-1] == len(flags) and np.all(np.diff(fo) >= 0)
        st = batch.last_stats
        assert st["mode"] == "match_mask_stream" and st["released"] == len(flags)
        for i in range(n):
            r_old = max(0, fed_bytes[i] - u.halo)
            fed_bytes[i] += u.unit * len(chunks[i])
            r_new = fed_bytes[i] if last[i] else max(0, fed_bytes[i] - u.halo)
            first, end = -(-r_old // u.unit), -(-r_new // u.unit)
            assert fs[i] == first and fo[i + 1] - fo[i] == end - first, (i, fed_bytes[i])
            assert first == len(got[i])
            got[i] += flags[fo[i]:fo[i + 1]].tolist()
            if cur[i] < len(queues[i]):
                ref = refs[i][cur[i]]
                assert got[i] == ref[:len(got[i])].tolist(), (i, cur[i], pos[i])
            if last[i]:
                assert got[i] == refs[i][cur[i]].tolist()
                got[i], pos[i], fed_bytes[i] = [], 0, 0
                cur[i] += 1
                done += 1
    return done


def ragged_queues(rng, n, alphabet, pats, per_slot=2, max_len=160):
    """Per slot, `per_slot` sequences of symbols of `alphabet` (each a list of units), some with a pattern planted."""
    queues = []
    for _ in range(n):
        q = []
        for _ in range(per_slot):
            pick = rng.integers(0, len(alphabet), size=int(rng.integers(0, max_len))) if rng.random() > 0.05 else []
            h = [x for j in pick for x in alphabet[j]]
            if h and rng.random() < 0.5:
                at = int(rng.integers(0, len(h) + 1))
                h = h[:at] + list(pats[int(rng.integers(0, len(pats)))]) * 3 + h[at:]
            q.append(np.asarray(h, dtype=np.int64))
        queues.append(q)
    return queues


def run_all(u, overlapping, queues, rng, step_max, batch=None, pattern_sets=None, set_index=None):
    u.overlapping = overlapping
    flat = [s for q in queues for s in q]
    idx = None
    if set_index is not None:   # each sequence searched with its slot's set
        idx = torch.tensor([int(set_index[i]) for i, q in enumerate(queues) for _ in q], dtype=set_index.dtype, device="cuda")
    ref = u.reference(flat, pattern_sets, idx)
    refs, at = [], 0
    for q in queues:
        refs.append(ref[at:at + len(q)])
        at += len(q)
    if batch is None:
        batch = u.ac.match_mask_stream_batch(len(queues), overlapping, pattern_sets=pattern_sets, set_index=set_index)
    return run_streams(u, batch, queues, rng, step_max, refs), batch


PATS = [b"abc", b"bcab", b"ca", b"abcabcaa", b"d", b"dd", b"bcd"]


def make(cls, kind, pats=PATS):
    if cls == "bytes":
        return Units(BytesAhoCorasick(pats, kind))
    if cls == "str":
        return Units(AhoCorasick([p.decode() for p in pats], kind))
    ids = [[int(b) * 300 for b in p] for p in pats]   # (below 2^16: uint16 ids too)
    return Units(TokenAhoCorasick(ids, kind), TOKEN_DTYPES[int(cls[-1])])


def alphabet(cls):
    """Symbols, each a list of units: for str 1-, 2- and 3-byte characters, cut anywhere by the byte chunks."""
    if cls == "str":
        return [list(c.encode()) for c in "abcdé€"]
    if cls == "bytes":
        return [[c] for c in b"abcd"]
    return [[c * 300] for c in b"abcd"] + [[5]]


def pats_units(cls, pats=PATS):
    return [np.frombuffer(p, dtype=np.uint8) if cls in ("bytes", "str") else np.array([int(b) * 300 for b in p]) for p in pats]


CLASSES = ["bytes", "str", "tokens0", "tokens1", "tokens2"]


@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_ragged_streams_equal_the_one_shot_mask(search, cls):
    kind, overlapping = search
    rng = np.random.default_rng(10 * CLASSES.index(cls) + kind.value + 5 * overlapping)
    u = make(cls, kind)
    queues = ragged_queues(rng, 70, alphabet(cls), pats_units(cls))
    done, batch = run_all(u, overlapping, queues, rng, 23)
    assert done > 70
    # the same batch again: every slot starts from a released state
    run_all(u, overlapping, ragged_queues(rng, 70, alphabet(cls), pats_units(cls), per_slot=1), rng, 5, batch=batch)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_generation_loop_one_token_per_stream_per_feed(search):
    """Banned sequences of 2-8 tokens; every stream gets one id per feed, k - 1 ids are held back until `last`."""
    kind, overlapping = search
    rng = np.random.default_rng(3)
    banned = [list(rng.integers(0, 50, size=int(rng.integers(2, 9)))) for _ in range(40)]
    u = Units(TokenAhoCorasick(banned, kind), torch.int64)
    u.overlapping = overlapping
    queues = []
    for _ in range(128):
        seq = list(rng.integers(0, 50, size=60))
        for _ in range(3):
            at = int(rng.integers(0, 60))
            seq[at:at] = banned[int(rng.integers(0, len(banned)))]
        queues.append([np.asarray(seq, dtype=np.int64)])
    refs = [[r] for r in u.reference([q[0] for q in queues])]
    batch = u.ac.match_mask_stream_batch(128, overlapping)
    assert run_streams(u, batch, queues, rng, 1, refs, one_step=True, last_p=1.0) == 128


@pytest.mark.parametrize("cls", ["bytes", "str", "tokens1"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_pattern_sets(search, cls):
    kind, overlapping = search
    rng = np.random.default_rng(17)
    u = make(cls, kind)
    sets = [[0, 3], [1, 2, 5], [4], list(range(len(PATS)))]
    ps = u.ac.pattern_sets(sets)
    n = 40
    set_index = torch.tensor(rng.integers(0, len(sets), size=n), dtype=torch.int64, device="cuda")
    queues = ragged_queues(rng, n, alphabet(cls), pats_units(cls))
    run_all(u, overlapping, queues, rng, 17, pattern_sets=ps, set_index=set_index)
    # an index outside [0, n_sets) admits no pattern: all False (set through the internal filter, which does not check)
    batch = u.ac.match_mask_stream_batch(n, overlapping, pattern_sets=ps, set_index=set_index)
    inner = getattr(batch, "_batch", batch)
    bad = set_index.clone()
    bad[::2] = len(sets)
    bad[1::4] = -1
    inner._flt = (ps, bad)
    refs = [[np.zeros(len(s), dtype=bool) if i % 2 == 0 or i % 4 == 1 else None for s in q] for i, q in enumerate(queues)]
    good = [i for i in range(n) if not (i % 2 == 0 or i % 4 == 1)]
    u.overlapping = overlapping
    ref_good = u.reference([s for i in good for s in queues[i]], ps, torch.tensor([int(set_index[i]) for i in good for _ in queues[i]],
                                                                                  dtype=torch.int64, device="cuda"))
    at = 0
    for i in good:
        refs[i] = ref_good[at:at + len(queues[i])]
        at += len(queues[i])
    run_streams(u, batch, queues, rng, 17, refs)


@pytest.mark.parametrize("tuning", ["small-tasks", "ring-1"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_long_patterns_whose_tails_span_several_sieve_tasks(search, tuning):
    kind, overlapping = search
    rng = np.random.default_rng(29)
    long_pats = [bytes(rng.choice(np.frombuffer(b"ab", dtype=np.uint8), size=int(m)).astype(np.uint8)) for m in (300, 1100, 3000)]
    pats = long_pats + [b"ab", b"ba", b"aab"]
    with tuned(tuning):
        u = Units(BytesAhoCorasick(pats, kind))
        queues = [[np.frombuffer(bytes(rng.choice(np.frombuffer(b"ab", dtype=np.uint8), size=int(rng.integers(0, 3000))).astype(np.uint8))
                                 + long_pats[i % 3] + long_pats[(i + 1) % 3][:1500], dtype=np.uint8).astype(np.int64)] for i in range(12)]
        run_all(u, overlapping, queues, rng, 4000)
        assert u.ac._ac.last_stats["task_bytes"] == 512


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_one_byte_patterns_hold_nothing(search):
    kind, overlapping = search
    rng = np.random.default_rng(41)
    u = Units(BytesAhoCorasick([b"a", b"c"], kind))
    queues = ragged_queues(rng, 30, alphabet("bytes"), [np.frombuffer(b"a", dtype=np.uint8)])
    _, batch = run_all(u, overlapping, queues, rng, 9)
    assert batch.last_stats["held"] == 0


def _merge(parts):
    out = []
    for s, e in parts:
        if out and out[-1][1] == s:
            out[-1] = (out[-1][0], e)
        else:
            out.append((s, e))
    return out


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_host_forms_merge_to_match_spans(search):
    kind, overlapping = search
    rng = np.random.default_rng(53)
    sac = AhoCorasick(["é€a", "bé", "€", "abcabc", "cab"], kind)
    bac = BytesAhoCorasick([b"abc", b"bcab", b"ca", b"abcabcaa"], kind)
    tac = TokenAhoCorasick([[1, 2], [2, 3, 1], [5], [1, 2, 1, 2, 1]], kind)
    for case in range(12):
        text = "".join(rng.choice(list("abcé€"), size=int(rng.integers(0, 80))))
        hay = bytes(rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=int(rng.integers(0, 80))).astype(np.uint8))
        ids = [int(x) for x in rng.integers(1, 6, size=int(rng.integers(0, 80)))]
        for ac, seq in ((sac, text), (bac, hay), (tac, ids)):
            patterns = [0, 2, 3] if case % 3 == 2 else None
            s = ac.match_spans_stream(overlapping, patterns=patterns)
            cuts = sorted(int(x) for x in rng.integers(0, len(seq) + 1, size=int(rng.integers(0, 6))))
            parts, released = [], 0
            for a, b in zip([0] + cuts, cuts + [len(seq)]):
                got = s.feed(seq[a:b])
                assert all(released <= x < y <= s.released for x, y in got)
                released = s.released
                parts += got
            parts += s.finish()
            assert s.released == len(seq)
            want = ac.match_spans(seq, overlapping, patterns=patterns)
            assert _merge(parts) == want, (type(ac).__name__, seq, cuts)


def test_two_threads_each_with_its_own_batch():
    errors = []

    def work(seed):
        try:
            rng = np.random.default_rng(seed)
            for cls, (kind, overlapping) in (("bytes", SEARCHES[2]), ("tokens2", SEARCHES[3])):
                u = make(cls, kind)
                run_all(u, overlapping, ragged_queues(rng, 50, alphabet(cls), pats_units(cls)), rng, 19)
        except Exception as e:   # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(s,)) for s in (1, 2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
