"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI
(include/acb200.h) by the package, against the CPU oracle on the same seeded
inputs, against the reference's golden vectors, and -- at larger sizes --
through size-independent properties.  Bit-exact: integer/index work."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, Implementation, MatchKind, workloads as W
from oracle import Oracle

from .gpu_helpers import KINDS, check_batch, dev, gpu_batch, kernel, set_kernel  # noqa: F401 (kernel: the fixture)

HERE = os.path.dirname(os.path.abspath(__file__))

with open(os.path.join(HERE, "golden", "reference_vectors.json"), encoding="utf-8") as f:
    VECTORS = json.load(f)["vectors"]


# ---------------------------------------------------------------- golden vectors, through the drop-in classes
@pytest.mark.parametrize("vec", VECTORS, ids=[f"{i}:{v['src']}" for i, v in enumerate(VECTORS)])
def test_reference_vectors(vec, kernel):
    kind = MatchKind[vec["kind"]]
    hay = vec["haystack"]
    if vec["cls"] == "str":
        ac = AhoCorasick(vec["patterns"], matchkind=kind)
        if vec.get("error"):
            with pytest.raises(ValueError):
                ac.find_matches_as_indexes(hay, overlapping=True)
            with pytest.raises(ValueError):
                ac.find_matches_as_strings(hay, overlapping=True)
            return
        idx = ac.find_matches_as_indexes(hay, overlapping=vec["overlapping"])
        if "expect_strings" in vec:
            assert [hay[s:e] for (_, s, e) in idx] == vec["expect_strings"]
            assert ac.find_matches_as_strings(hay, overlapping=vec["overlapping"]) == vec["expect_strings"]
    else:
        raw = hay.encode()
        ac = BytesAhoCorasick([p.encode() for p in vec["patterns"]], matchkind=kind)
        if vec.get("error"):
            with pytest.raises(ValueError):
                ac.find_matches_as_indexes(raw, overlapping=True)
            return
        idx = ac.find_matches_as_indexes(raw, overlapping=vec["overlapping"])
        if "expect_strings" in vec:
            assert [raw[s:e].decode() for (_, s, e) in idx] == vec["expect_strings"]
    if "expect_indexes" in vec:
        assert [list(t) for t in idx] == vec["expect_indexes"]
    assert all(isinstance(x, int) for t in idx for x in t)


# ---------------------------------------------------------------- seeded batches vs the oracle
@pytest.mark.parametrize("kind", KINDS, ids=lambda k: k.name)
def test_ragged_small_alphabet(kind, kernel):
    rng = np.random.default_rng(11)
    pats = sorted({bytes(rng.integers(97, 100, size=rng.integers(1, 6)).astype(np.uint8)) for _ in range(40)})
    pats += pats[:3]  # duplicates: distinct ids, same string
    data, offs = W.ragged(3000, 300, b"abc", seed=12)
    n = check_batch(pats, kind, data, offs)
    assert n > 1000
    if kind == MatchKind.Standard:
        check_batch(pats, kind, data, offs, overlapping=True)


@pytest.mark.parametrize("kind", KINDS, ids=lambda k: k.name)
def test_config2_shape_scaled(kind, kernel):
    pats, data, offs = W.config2(1500)
    n = check_batch([p.encode() for p in pats], kind, data, offs, codepoints=True, implementation=Implementation.DFA)
    assert n > 50


@pytest.mark.parametrize("kind", KINDS, ids=lambda k: k.name)
def test_config3_shape_scaled(kind, kernel):
    pats, data, offs = W.config3(n_patterns=2000, n_lines=4000)
    n = check_batch(pats, kind, data, offs)
    assert n > 1000


def test_config5_shape_scaled(kernel):
    pats, data, offs = W.config5(n_patterns=20000, n_haystacks=512, hay_bytes=4096)
    check_batch(pats, MatchKind.Standard, data, offs)


def test_config4_shape_scaled_chunked_overlapping(kernel):
    pats, data = W.config4(n_patterns=20000, hay_bytes=3_000_017)
    orc = Oracle(pats, "Standard")
    exp = orc.find(data.tobytes(), overlapping=True)
    ac = BytesAhoCorasick(pats, implementation=Implementation.ContiguousNFA)
    m, moffs, total = ac.scan_device(dev(data), dev(np.array([0, len(data)], dtype=np.int64)), overlapping=True)
    got = m.cpu().numpy().view(np.uint32)
    assert total == len(exp) and moffs.tolist() == [0, total]
    assert [tuple(int(x) for x in r[1:]) for r in got] == exp
    # the drop-in call takes the same path for a large haystack
    assert ac.find_matches_as_indexes(data.tobytes(), overlapping=True) == exp


@pytest.mark.parametrize("kind", KINDS, ids=lambda k: k.name)
def test_one_large_haystack_non_overlapping(kind, kernel):
    """One multi-megabyte haystack, non-overlapping: segments of the SAME haystack are scanned in
    parallel from speculated states and must still give the serial (restart-at-match-end) answer."""
    rng = np.random.default_rng(21)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 7)).astype(np.uint8)) for _ in range(300)})
    data = rng.integers(97, 101, size=1_500_003, dtype=np.uint8).astype(np.uint8)
    exp = Oracle(pats, kind.name).find(data.tobytes())
    assert len(exp) > 10_000
    ac = BytesAhoCorasick(pats, kind)
    assert ac.find_matches_as_indexes(data.tobytes()) == exp
    if kernel not in ("plain", "sieve", "sieve-small-tasks"):
        assert ac._ac.last_stats["segments"] > 1000


def test_dense_self_overlapping_matches_single_haystack(kernel):
    """'aa' on a run of 'a' at an odd offset: every guessed restart phase is wrong and the
    repair pass has to carry the truth through the whole haystack."""
    for lead in (1, 2):
        hay = b"b" * lead + b"a" * 20_001
        exp = Oracle([b"aa"], "Standard").find(hay)
        assert BytesAhoCorasick([b"aa"]).find_matches_as_indexes(hay) == exp


def test_unaligned_base_and_tiny_haystacks(kernel):
    pats = [b"ab", b"b", b"abab", b"ba"]
    rng = np.random.default_rng(5)
    body = rng.integers(97, 99, size=5000, dtype=np.uint8).astype(np.uint8)
    for shift in (1, 7, 33):
        lens = rng.integers(0, 40, size=200)
        offs = np.zeros(201, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        offs += shift
        for kind in KINDS:
            orc = Oracle(pats, kind.name)
            total, counts, rec = orc.scan_batch(body, offs)
            ac = BytesAhoCorasick(pats, kind)
            m, moffs, gtotal = gpu_batch(ac, body, offs)
            assert gtotal == total and np.array_equal(m, rec)


def test_implementations_agree(kernel):
    hay = "hello, world, hello again ☃ héllo"
    pats = ["hello", "world", "☃ h", "llo"]
    res = [AhoCorasick(pats, implementation=i).find_matches_as_indexes(hay, overlapping=True)
           for i in (None, Implementation.NoncontiguousNFA, Implementation.ContiguousNFA, Implementation.DFA)]
    assert all(r == res[0] for r in res) and len(res[0]) >= 4


def test_output_capacity_retry():
    pats = [b"a"]
    data = np.full(50_000, 97, dtype=np.uint8)
    offs = np.array([0, 50_000], dtype=np.int64)
    ac = BytesAhoCorasick(pats)
    m, moffs, total = ac.scan_device(dev(data), dev(offs), capacity=1024)
    assert total == 50_000 and moffs.tolist() == [0, 50_000]
    got = m.cpu().numpy().view(np.uint32)
    assert np.array_equal(got[:, 2], np.arange(50_000)) and np.array_equal(got[:, 3], np.arange(1, 50_001))


# ---------------------------------------------------------------- full-size properties (no oracle at this size)
def test_full_size_properties_config2():
    """BASELINE config 2 at full size: sharding invariance (scan of the batch ==
    concatenation of scans of its halves), every hit slices back to its pattern,
    and the known structure of the workload (only i % 90 == 0 haystacks carry names)."""
    pats, data, offs = W.config2(20_000)
    ac = AhoCorasick(pats, implementation=Implementation.DFA)
    d, o = dev(data), dev(offs)
    m, moffs, total = ac.scan_device(d, o)
    m = m.cpu().numpy().view(np.uint32).copy()
    moffs = moffs.cpu().numpy().copy()
    half = 10_000
    m1, o1, t1 = ac.scan_device(d[: offs[half]], o[: half + 1].clone())
    m1 = m1.cpu().numpy().view(np.uint32).copy()
    m2, o2, t2 = ac.scan_device(d[offs[half]:], dev(offs[half:] - offs[half]))
    m2 = m2.cpu().numpy().view(np.uint32).copy()
    m2[:, 0] += half
    assert t1 + t2 == total and np.array_equal(np.concatenate([m1, m2]), m)
    # plain kernel agrees with the staged kernel
    set_kernel(1)
    try:
        mp, _, tp = ac.scan_device(d, o)
        assert tp == total and np.array_equal(mp.cpu().numpy().view(np.uint32), m)
    finally:
        set_kernel(0)
    hays_with = np.unique(m[:, 0])
    assert len(hays_with) > 0 and np.all(hays_with % 90 == 0)
    for h, pid, s, e in m[:200]:
        text = data[offs[h]:offs[h + 1]].tobytes().decode("utf-8")
        assert text[s:e] == pats[pid]


# ---------------------------------------------------------------- inputs above one call's 32-bit range (cut up on the host)
def test_windows_and_runs_match_one_call(monkeypatch):
    """The windowing used for buffers above 2 GiB, exercised at a small limit: a batch is cut into runs of whole
    haystacks, a single large haystack (overlapping search) into windows sharing max_pattern_len - 1 bytes."""
    from ahocorasick_rs_b200 import matcher
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    # (a) a ragged batch, all kinds
    data, offs = W.ragged(400, 3000, b"abcd", seed=32)
    for kind in KINDS:
        ac = BytesAhoCorasick(pats, kind)
        m0, o0, t0 = ac.scan_device(dev(data), dev(offs))
        m0, o0 = m0.clone(), o0.clone()  # (views of the automaton's workspace: the next call reuses it)
        monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
        m1, o1, t1 = ac.scan_device(dev(data), dev(offs))
        monkeypatch.undo()
        assert t1 == t0 and m1.dtype == torch.int64
        assert np.array_equal(m1.cpu().numpy(), m0.cpu().numpy().view(np.uint32).astype(np.int64))
        assert np.array_equal(o1.cpu().numpy(), o0.cpu().numpy().astype(np.int64))
    # (b) one large haystack, overlapping, bytes and code points (multi-byte characters straddling window cuts)
    hay = rng.integers(97, 101, size=400_000, dtype=np.uint8).astype(np.uint8)
    exp = Oracle(pats, "Standard").find(hay.tobytes(), overlapping=True)
    ac = BytesAhoCorasick(pats)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 30_001)
    got = ac.find_matches_as_indexes(hay.tobytes(), overlapping=True)
    # non-overlapping on a single oversized haystack: selected from the windows' overlapping lists, every match kind
    non = {kind: BytesAhoCorasick(pats, kind).find_matches_as_indexes(hay.tobytes()) for kind in KINDS}
    monkeypatch.undo()
    assert got == exp
    for kind in KINDS:
        assert non[kind] == Oracle(pats, kind.name).find(hay.tobytes()), kind
    text = "".join(rng.choice(list("ab—é☃cd"), size=60_000))
    upats = ["a—", "—é", "☃c", "b", "é☃c", "dd"]
    ref = AhoCorasick(upats).find_matches_as_indexes(text, overlapping=True)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 9_973)
    got = AhoCorasick(upats).find_matches_as_indexes(text, overlapping=True)
    monkeypatch.undo()
    assert got == ref and len(ref) > 10_000
    assert ref == [(p, s, e) for (p, s, e) in Oracle([u.encode() for u in upats], "Standard").find_str(text, overlapping=True)]


# ---------------------------------------------------------------- the reference's property tests, through the drop-in classes
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=60, deadline=None)
@given(st.text(), st.text(min_size=1), st.text(), st.sampled_from([True, False, None]))
def test_unicode_extensive_like_the_reference(prefix, pattern, suffix, store_patterns):
    """reference tests/test_ac.py:135-154: one arbitrary unicode pattern inside arbitrary text; every hit slices back
    to the pattern, and the first hit is where str.find puts it."""
    haystack = prefix + pattern + suffix
    ac = AhoCorasick([pattern]) if store_patterns is None else AhoCorasick([pattern], store_patterns=store_patterns)
    idx = ac.find_matches_as_indexes(haystack)
    assert {i for (i, _, _) in idx} == {0}
    assert {haystack[s:e] for (_, s, e) in idx} == {pattern}
    assert set(ac.find_matches_as_strings(haystack)) == {pattern}
    assert idx[0][1] == haystack.find(pattern)


@settings(max_examples=25, deadline=None)
@given(st.lists(st.text(min_size=3), min_size=1, max_size=300), st.sampled_from([True, False, None]))
def test_construction_extensive_like_the_reference(patterns, store_patterns):
    """reference tests/test_ac.py:86-100 (pattern lists scaled down from 30 000 to 300 per example: every
    call here is a GPU round trip; the 30 000-pattern construction itself is in the CPU tests)."""
    patterns = [f"{p}_{i}_" for (i, p) in enumerate(patterns)]
    ac = AhoCorasick(patterns, store_patterns=store_patterns)
    for p in patterns[:40]:
        assert ac.find_matches_as_strings(p) == [p]


@settings(max_examples=40, deadline=None)
@given(st.binary(), st.binary(min_size=1), st.binary())
def test_bytes_extensive_like_the_reference(prefix, pattern, suffix):
    """reference tests/test_ac_bytes.py:133-161: arbitrary bytes, including 0x00 and 0xff."""
    haystack = prefix + pattern + suffix
    idx = BytesAhoCorasick([pattern]).find_matches_as_indexes(haystack)
    assert {i for (i, _, _) in idx} == {0}
    assert {haystack[s:e] for (_, s, e) in idx} == {pattern}
    assert idx[0][1] == haystack.find(pattern)
