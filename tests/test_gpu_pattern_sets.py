"""Pattern sets on the device: every covered query of the three classes against the CPU oracle built from each
haystack's (or stream's) subset of the patterns, with the ids mapped back to the full automaton."""
import random

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick
from ahocorasick_rs_b200.matcher import _Automaton
from oracle import Oracle

pytestmark = pytest.mark.gpu

KINDS = [MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest]
SEARCHES = [(k, False) for k in KINDS] + [(MatchKind.Standard, True)]
SEARCH_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest", "Overlapping"]


def subset_find(patterns, S, hay: bytes, kind, overlapping=False):
    """The oracle's rows for an automaton of only the patterns in S (same order), ids mapped back."""
    ids = sorted(S)
    if not ids:
        return []
    o = Oracle([patterns[i] for i in ids], kind.value)
    return [(ids[p], s, e) for p, s, e in o.find(hay, overlapping)]


def _cp(hay: bytes, rows):
    """byte rows -> code point rows of UTF-8 text"""
    def cp(i):
        return len(hay[:i].decode("utf-8"))
    return [(p, cp(s), cp(e)) for p, s, e in rows]


def _batch(hays, dev):
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    data = torch.from_numpy(np.frombuffer(b"".join(hays) or b"\0", dtype=np.uint8)[:offs[-1]].copy()).to(dev)
    return data, torch.from_numpy(offs).to(dev)


def _random_case(seed, n_hay=40, alpha=b"abcd"):
    rng = random.Random(seed)
    pats = [bytes(rng.choice(alpha) for _ in range(rng.randint(1, 6))) for _ in range(30)]
    pats += [pats[3], pats[3], b"abcd", b"bcd", b"cd"]   # duplicates, a nested family
    hays = [bytes(rng.choice(alpha) for _ in range(rng.choice([0, 1, 5, 50, 300, 2000]))) for _ in range(n_hay)]
    P = len(pats)
    sets = [[], list(range(P))] + [[p for p in range(P) if rng.random() < f] for f in (0.05, 0.2, 0.5, 0.9)]
    idx = [rng.randrange(len(sets)) for _ in hays]
    return pats, hays, sets, idx


def _rows(m, mo, n):
    m, mo = m.cpu().numpy().astype(np.int64), mo.cpu().numpy()
    return [[tuple(int(x) for x in r[1:4]) for r in m[mo[i]:mo[i + 1]]] for i in range(n)]


@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_device_queries_bytes(kind, overlapping, seed, idx_dtype):
    dev = torch.device("cuda")
    pats, hays, sets, idx = _random_case(seed)
    ac = BytesAhoCorasick(pats, matchkind=kind)
    ps = ac.pattern_sets(sets)
    si = torch.tensor(idx, dtype=idx_dtype, device=dev)
    data, offs = _batch(hays, dev)
    want = [subset_find(pats, sets[idx[i]], h, kind, overlapping) for i, h in enumerate(hays)]
    m, mo, _ = ac.scan_device(data, offs, overlapping, pattern_sets=ps, set_index=si)
    assert _rows(m, mo, len(hays)) == want
    assert ac._ac.last_stats["engine"] == "sieve" and ac._ac.last_stats["pattern_sets"] == len(sets)
    counts = ac.count_matches_device(data, offs, overlapping, pattern_sets=ps, set_index=si).tolist()
    assert counts == [len(w) for w in want]
    if not overlapping:
        first = ac.find_first_device(data, offs, pattern_sets=ps, set_index=si).tolist()
        assert [tuple(r) if r[0] >= 0 else None for r in first] == [w[0] if w else None for w in want]
        anym = ac.is_match_device(data, offs, pattern_sets=ps, set_index=si).tolist()
        assert anym == [bool(w) for w in want]


@pytest.mark.parametrize("kind", KINDS)
def test_full_set_equals_unfiltered(kind):
    dev = torch.device("cuda")
    pats, hays, _, _ = _random_case(7)
    ac = BytesAhoCorasick(pats, matchkind=kind)
    ps = ac.pattern_sets([range(len(pats))])
    si = torch.zeros(len(hays), dtype=torch.int32, device=dev)
    data, offs = _batch(hays, dev)
    m0, mo0, t0 = ac.scan_device(data, offs)
    m0, mo0 = m0.clone(), mo0.clone()
    m1, mo1, t1 = ac.scan_device(data, offs, pattern_sets=ps, set_index=si)
    assert t0 == t1 and torch.equal(m0, m1) and torch.equal(mo0, mo1)
    assert torch.equal(ac.find_first_device(data, offs), ac.find_first_device(data, offs, pattern_sets=ps, set_index=si))
    assert torch.equal(ac.is_match_device(data, offs), ac.is_match_device(data, offs, pattern_sets=ps, set_index=si))
    assert torch.equal(ac.count_matches_device(data, offs), ac.count_matches_device(data, offs, pattern_sets=ps, set_index=si))


@pytest.mark.parametrize("kind", KINDS)
def test_duplicates_and_nested_family(kind):
    pats = [b"stop", b"stop", b"stop", b"xstop", b"top", b"op"]
    ac = BytesAhoCorasick(pats, matchkind=kind)
    hay = b"..xstop.."
    for S in ([1, 2], [2], [4, 5], [5], [0, 5], []):
        want = subset_find(pats, S, hay, kind)
        assert ac.find_matches_as_indexes(hay, patterns=S) == want
        assert ac.find_first(hay, patterns=S) == (want[0] if want else None)
        assert ac.is_match(hay, patterns=S) == bool(want)
        assert ac.count_matches(hay, patterns=S) == len(want)


@pytest.mark.parametrize("kind", KINDS)
def test_host_batches_str(kind):
    rng = random.Random(3)
    words = ["héllo", "wörld", "日本", "日本語", "語", "a", "ab", "🎉x"]
    ac = AhoCorasick(words, matchkind=kind)
    hays = ["".join(rng.choice(words + [" ", "z"]) for _ in range(rng.randint(0, 30))) for _ in range(25)]
    sets = [[p for p in range(len(words)) if rng.random() < 0.5] for _ in hays]
    pb = [w.encode() for w in words]
    want = [_cp(h.encode(), subset_find(pb, S, h.encode(), kind)) for h, S in zip(hays, sets)]
    assert ac.find_matches_as_indexes_batch(hays, patterns=sets) == want
    assert ac.find_first_batch(hays, patterns=sets) == [w[0] if w else None for w in want]
    assert ac.is_match_batch(hays, patterns=sets) == [bool(w) for w in want]
    assert ac.count_matches_batch(hays, patterns=sets) == [len(w) for w in want]
    assert ac.find_matches_as_indexes(hays[0], patterns=sets[0]) == want[0]
    strs = ac.find_matches_as_strings(hays[1], patterns=sets[1])
    assert strs == [words[p] for p, _, _ in want[1]]


def test_overlapping_str_device():
    words = ["ab", "b", "bé", "é"]
    ac = AhoCorasick(words)
    hays = ["abé" * 3, "", "béab"]
    data, offs = _batch([h.encode() for h in hays], torch.device("cuda"))
    ps = ac.pattern_sets([[1, 2], [0]])
    si = torch.tensor([0, 1, 1], device="cuda")
    m, mo, _ = ac.scan_device(data, offs, True, pattern_sets=ps, set_index=si)
    pb = [w.encode() for w in words]
    want = [_cp(h.encode(), subset_find(pb, [[1, 2], [0]][s], h.encode(), MatchKind.Standard, True)) for h, s in zip(hays, [0, 1, 1])]
    assert _rows(m, mo, 3) == want


@pytest.mark.parametrize("kind", KINDS)
def test_windowed_paths(kind, monkeypatch):
    """WINDOW_BYTES patched small: runs of whole haystacks and one haystack above the limit, each with its own set."""
    monkeypatch.setattr(_Automaton, "WINDOW_BYTES", 4096)
    rng = random.Random(11)
    pats = [b"needle", b"need", b"le", b"eedl", b"xyz"]
    hays = [bytes(rng.choice(b"needlxyz ") for _ in range(n)) for n in (100, 3000, 9000, 50, 0, 2500)]
    sets = [[0], [1, 2], [2, 3], [], [0, 1, 2, 3, 4]]
    idx = [0, 1, 2, 4, 3, 1]
    dev = torch.device("cuda")
    ac = BytesAhoCorasick(pats, matchkind=kind)
    ps = ac.pattern_sets(sets)
    si = torch.tensor(idx, device=dev)
    data, offs = _batch(hays, dev)
    want = [subset_find(pats, sets[idx[i]], h, kind) for i, h in enumerate(hays)]
    m, mo, _ = ac.scan_device(data, offs, pattern_sets=ps, set_index=si)
    assert _rows(m, mo, len(hays)) == want
    assert ac.count_matches_device(data, offs, pattern_sets=ps, set_index=si).tolist() == [len(w) for w in want]
    first = ac.find_first_device(data, offs, pattern_sets=ps, set_index=si).tolist()
    assert [tuple(r) if r[0] >= 0 else None for r in first] == [w[0] if w else None for w in want]
    assert ac.is_match_device(data, offs, pattern_sets=ps, set_index=si).tolist() == [bool(w) for w in want]
    if kind == MatchKind.Standard:
        want_o = [subset_find(pats, sets[idx[i]], h, kind, True) for i, h in enumerate(hays)]
        m, mo, _ = ac.scan_device(data, offs, True, pattern_sets=ps, set_index=si)
        assert _rows(m, mo, len(hays)) == want_o
        assert ac.count_matches_device(data, offs, True, pattern_sets=ps, set_index=si).tolist() == [len(w) for w in want_o]


def test_text_that_picks_a_table_walker_runs_the_sieve_filtered(monkeypatch):
    """Config-2-like text, whose unfiltered scan the engine rule gives to a table walker: a filtered call is the sieve."""
    from ahocorasick_rs_b200 import workloads
    monkeypatch.setattr(_Automaton, "AUTO_PROFILE_BYTES", 1 << 16)
    names, data_np, offs_np = workloads.config2(n_haystacks=360, hay_bytes=4096)
    pats = [p.encode() for p in names]
    dev = torch.device("cuda")
    ac = BytesAhoCorasick(pats)
    data, offs = torch.from_numpy(data_np).to(dev), torch.from_numpy(offs_np).to(dev)
    ac.scan_device(data, offs)
    assert ac._ac.last_stats["engine"] == "table"
    sets = [list(range(0, len(pats), 2)), list(range(len(pats)))]
    n = offs_np.size - 1
    si = torch.tensor([i % 2 for i in range(n)], device=dev)
    m, mo, _ = ac.scan_device(data, offs, pattern_sets=ac.pattern_sets(sets), set_index=si)
    assert ac._ac.last_stats["engine"] == "sieve"
    got = _rows(m, mo, n)
    for i in range(0, n, 7):
        hay = data_np[offs_np[i]:offs_np[i + 1]].tobytes()
        assert got[i] == subset_find(pats, sets[i % 2], hay, MatchKind.Standard)


@pytest.mark.parametrize("kind", KINDS)
def test_byte_streams_per_stream_sets(kind):
    rng = random.Random(5)
    pats = [b"stop", b"op", b"halt", b"st", b"alt"]
    n = 12
    sets = [[0], [1, 3], [2], [], [0, 1, 2, 3, 4]]
    idx = [rng.randrange(len(sets)) for _ in range(n)]
    streams = [bytes(rng.choice(b"stophal ") for _ in range(rng.randint(0, 80))) for _ in range(n)]
    ac = BytesAhoCorasick(pats, matchkind=kind)
    ps = ac.pattern_sets(sets)
    si = torch.tensor(idx, device="cuda")
    im = ac.is_match_stream_batch(n, pattern_sets=ps, set_index=si)
    ff = ac.find_first_stream_batch(n, pattern_sets=ps, set_index=si)
    pos = [0] * n
    last = None
    for step in range(12):
        chunks = []
        for i in range(n):
            k = rng.randint(0, 9)
            chunks.append(streams[i][pos[i]:pos[i] + k])
            pos[i] += k
        final = step == 11
        if final:
            chunks = [streams[i][pos[i] - len(chunks[i]):] for i in range(n)]
        data, offs = _batch(chunks, torch.device("cuda"))
        lt = torch.ones(n, dtype=torch.bool, device="cuda") if final else None
        flags = im.feed_device(data, offs, lt).tolist()
        rows = ff.feed_device(data, offs, lt).tolist()
        last = flags, rows
    flags, rows = last
    for i in range(n):
        want = subset_find(pats, sets[idx[i]], streams[i], kind)
        assert flags[i] == bool(want)
        assert (tuple(rows[i]) if rows[i][0] >= 0 else None) == (want[0] if want else None)


def test_single_query_streams():
    ac = AhoCorasick(["fin", "finé", "né"], matchkind=MatchKind.LeftmostLongest)
    s = ac.find_first_stream(patterns=[2])
    s.feed("xxfi")
    s.feed("né")
    want = _cp("xxfiné".encode(), subset_find([w.encode() for w in ["fin", "finé", "né"]], [2], "xxfiné".encode(), MatchKind.LeftmostLongest))
    assert s.finish() == want[0]
    m = ac.is_match_stream(patterns=[0])
    assert m.feed("xxf") is False
    assert m.feed("inx") is True


@pytest.mark.parametrize("kind", KINDS)
def test_token_stop_sequences(kind):
    """Per-request stop sequences during batched generation: one token per stream per feed, stop sequences split
    across feeds, each stream with its own set."""
    rng = random.Random(9)
    stops = [[50256], [13, 13], [198, 198, 198], [7, 8, 9, 10], [8, 9], [1000, 2000]]
    ac = TokenAhoCorasick(stops, matchkind=kind)
    n = 64
    sets = [[0], [1, 2], [3], [4], [3, 4], [5], [], list(range(len(stops)))]
    idx = [rng.randrange(len(sets)) for _ in range(n)]
    vocab = [13, 198, 7, 8, 9, 10, 1000, 2000, 5, 6, 50256]
    streams = [[rng.choice(vocab) for _ in range(rng.randint(1, 40))] for _ in range(n)]
    ps = ac.pattern_sets(sets)
    ff = ac.find_first_stream_batch(n, pattern_sets=ps, set_index=torch.tensor(idx, device="cuda"))
    T = max(len(s) for s in streams)
    for t in range(T + 1):
        final = t == T
        chunk = [s[t:t + 1] if not final else [] for s in streams]
        toks = torch.tensor([x for c in chunk for x in c] or [0], dtype=torch.int64, device="cuda")[:sum(len(c) for c in chunk)]
        offs = torch.tensor(np.concatenate([[0], np.cumsum([len(c) for c in chunk])]), dtype=torch.int64, device="cuda")
        rows = ff.feed_device(toks, offs, torch.ones(n, dtype=torch.bool, device="cuda") if final else None)
    rows = rows.tolist()
    enc = lambda seq: b"".join(bytes([0x80 | (x >> 14), (x >> 7) & 0x7F, x & 0x7F]) for x in seq)
    for i in range(n):
        want = subset_find([enc(s) for s in stops], sets[idx[i]], enc(streams[i]), kind)
        want = (want[0][0], want[0][1] // 3, want[0][2] // 3) if want else None
        assert (tuple(rows[i]) if rows[i][0] >= 0 else None) == want, i
    # the device and host query forms on the same ids
    hays = streams[:8]
    got = ac.find_first_batch(hays, patterns=[sets[idx[i]] for i in range(8)])
    for i in range(8):
        want = subset_find([enc(s) for s in stops], sets[idx[i]], enc(hays[i]), kind)
        assert got[i] == ((want[0][0], want[0][1] // 3, want[0][2] // 3) if want else None)
