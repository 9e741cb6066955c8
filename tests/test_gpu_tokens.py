"""GPU tests of TokenAhoCorasick (-m gpu): the encode kernel against the host encoder and the numpy statement of the
format (every id width, every tail length, misaligned views, bad-id reports); search parity on every kernel variant and
search, against the oracle on the encoded bytes divided by 3 and against a token-level brute force; every device query
and its host batch form; a batch whose encoding exceeds WINDOW_BYTES; the stream search and the stream queries against
the stream models; a stop-sequence batch fed one token per step; two threads on one object."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import MatchKind, TokenAhoCorasick, _capi  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, VARIANTS, forced  # noqa: E402
from .stream_model import released_by  # noqa: E402
from .stream_query_model import expected  # noqa: E402
from .test_tokens_cpu import NO_BAD, host_encode, numpy_format  # noqa: E402

DTYPES = {torch.int32: 4, torch.int64: 8, torch.uint16: 2}
# ids that share low bytes (t, t + 2^7, t + 2^14), the edges of each byte, 0 (80 00 00) and the largest id
ALPHA = [0, 1, 127, 128, 5, 5 + (1 << 7), 5 + (1 << 14), 1 << 14, (1 << 14) + 1, 1 + (1 << 7), (1 << 21) - 1]


def enc(ids):
    return numpy_format(ids).tobytes()


def tok_brute(pats, hay, kind, overlapping):
    """The token-level statement, over lists: every occurrence, then the kind's selection (SURVEY.md §8c)."""
    occ = [(p, i, i + len(q)) for p, q in enumerate(pats) for i in range(len(hay) - len(q) + 1) if hay[i:i + len(q)] == q]
    if overlapping:
        return sorted(occ, key=lambda m: (m[2], m[1], m[0]))
    key = {MatchKind.Standard: lambda m: (m[2], m[1], m[0]), MatchKind.LeftmostFirst: lambda m: (m[1], m[0]),
           MatchKind.LeftmostLongest: lambda m: (m[1], -m[2], m[0])}[kind]
    out, s = [], 0
    while True:
        c = [m for m in occ if m[1] >= s]
        if not c:
            return out
        m = min(c, key=key)
        out.append(m)
        s = m[2]


def oracle_rows(pats, hays, kind, overlapping):
    """Per haystack, the oracle's rows on the encoded bytes with positions divided by 3."""
    orc = Oracle([enc(p) for p in pats], kind.name)
    out = []
    for h in hays:
        rows = orc.find(enc(h), overlapping=overlapping)
        assert all(s % 3 == 0 and e % 3 == 0 for _, s, e in rows)
        out.append([(p, s // 3, e // 3) for p, s, e in rows])
    return out


def device_batch(hays, dtype=torch.int32, shift=0):
    """The haystacks as one 1-D CUDA tensor of ids, `shift` elements past an aligned allocation, and int64 offsets."""
    lens = [len(h) for h in hays]
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    np_dtype = {torch.int32: np.int32, torch.int64: np.int64, torch.uint16: np.uint16}[dtype]
    flat = np.concatenate([np.asarray(h, dtype=np.int64) for h in hays]).astype(np_dtype) if offs[-1] else np.zeros(0, np_dtype)
    base = torch.empty(shift + len(flat) + 1, dtype=dtype, device="cuda")
    t = base[shift:shift + len(flat)]
    if len(flat):
        t.copy_(torch.from_numpy(flat))
    return t, torch.from_numpy(offs).cuda()


# ---------------------------------------------------------------- the encode kernel
def device_encode(t, out_shift=0):
    n = t.numel()
    out = torch.full((3 * n + out_shift + 1,), 0xEE, dtype=torch.uint8, device="cuda")
    bad = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = _capi.lib().acb_tokens_encode(t.data_ptr(), t.element_size(), n, out[out_shift:].data_ptr(), bad.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == _capi.ACB_OK, _capi.last_error()
    o = out.cpu().numpy()
    assert o[-1] == 0xEE and (out_shift == 0 or o[0] == 0xEE)
    return o[out_shift:-1], int(bad.item()) & NO_BAD


@pytest.mark.parametrize("dtype", list(DTYPES), ids=[str(d) for d in DTYPES])
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_encode_kernel_every_tail(dtype, shift):
    rng = np.random.default_rng(shift)
    hi = 1 << 16 if dtype == torch.uint16 else 1 << 21
    for n in range(68):
        ids = rng.integers(0, hi, n)
        ids[: min(n, 3)] = [hi - 1, 0, 128][: min(n, 3)]
        t = device_batch([ids.tolist()], dtype, shift)[0]
        got, bad = device_encode(t)
        assert bad == NO_BAD
        want = numpy_format(ids)
        assert np.array_equal(got, want), (n, shift)
        assert np.array_equal(got, host_encode(ids, DTYPES[dtype])[0])
    # the output off the 4-byte grid: the scalar path writes it
    ids = rng.integers(0, hi, 1000)
    got, _ = device_encode(device_batch([ids.tolist()], dtype, shift)[0], out_shift=1)
    assert np.array_equal(got, numpy_format(ids))


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["int32", "int64"])
@pytest.mark.parametrize("shift", [0, 1])
def test_encode_kernel_reports_first_bad_index(dtype, shift):
    ids = np.arange(1000) % 5000
    for where, value in ((999, -1), (996, 1 << 21), (517, -7), (8, (1 << 21) + 3), (0, -1)):
        ids[where] = value
        t = device_batch([ids.tolist()], dtype, shift)[0]
        assert device_encode(t)[1] == where
    if dtype == torch.int64:
        ids[0] = 1 << 62
        assert device_encode(device_batch([ids.tolist()], dtype, shift)[0])[1] == 0


def test_bad_ids_raise_and_the_next_call_works():
    ac = TokenAhoCorasick([[1, 2], [2, 3, 4]])
    good = [[0, 1, 2, 3, 4], [2, 3, 4, 1, 2]]
    t, offs = device_batch(good)
    want = ac.find_matches_as_indexes_batch(good)
    assert want == [[(0, 1, 3)], [(1, 0, 3), (0, 3, 5)]]   # [2, 3, 4] starts inside [1, 2] in haystack 0
    for bad_id in (-1, 1 << 21):
        bad, boffs = device_batch([[1, 2, 3], [4, bad_id, 1, 2]], torch.int64)
        for call in (ac.scan_device, ac.is_match_device, ac.find_first_device, ac.count_matches_device,
                     ac.count_matches_by_pattern_device, ac.matching_patterns_device):
            with pytest.raises(ValueError, match=rf"token 4 = {bad_id} is outside"):
                call(bad, boffs)
        m, mo, total = ac.scan_device(t, offs)
        m, mo = m.tolist(), mo.tolist()
        assert total == 3 and [[tuple(r[1:]) for r in m[mo[i]:mo[i + 1]]] for i in range(2)] == want
    sb = ac.find_first_stream_batch(2)
    with pytest.raises(ValueError, match="token 1 = -1"):
        sb.feed_device(torch.tensor([1, -1], dtype=torch.int32, device="cuda"), torch.tensor([0, 1, 2], device="cuda"))
    out = sb.feed_device(torch.tensor([1, 2, 2, 3, 4], dtype=torch.int32, device="cuda"), torch.tensor([0, 2, 5], device="cuda"))
    assert out.tolist() == [[0, 0, 2], [1, 0, 3]]


def test_offsets_outside_the_ids_raise_before_any_scan():
    """Token offsets are multiplied by 3: one that is negative or past the ids (which could wrap in int64, e.g.
    -6148914691236517205 * 3 == 1, and cut a token) raises ValueError before any device work."""
    ac = TokenAhoCorasick([[1, 2]])
    t, _ = device_batch([[1, 2, 1, 2]])
    for bad in ([0, 5], [-1, 4], [0, -6148914691236517205], [0, 3074457345618258603, 4], [0, (1 << 63) - 1]):
        offs = torch.tensor(bad, dtype=torch.int64, device="cuda")
        for call in (ac.scan_device, ac.is_match_device, ac.find_first_device, ac.count_matches_device,
                     ac.count_matches_by_pattern_device, ac.matching_patterns_device, ac.stream_batch(len(bad) - 1).feed_device):
            with pytest.raises(ValueError, match=r"offsets must lie in \[0, 4\]"):
                call(t, offs)
    m, mo, total = ac.scan_device(t, torch.tensor([0, 1, 4], dtype=torch.int64, device="cuda"))
    assert total == 1 and m[:, 1:].tolist() == [[0, 1, 3]] and mo.tolist() == [0, 0, 1]


def test_scan_device_guards_the_workspace_it_copies_from():
    """scan_device copies its rows out of the automaton's workspace slot 0 and records the event that the next scan
    on that slot waits for (any thread, any stream), as first_device does."""
    pats, hays = parity_case(43)
    ac = TokenAhoCorasick(pats)
    t, offs = device_batch(hays)
    m, mo, total = ac.scan_device(t, offs)
    ws = ac._ac._ws[(t.device.index, 0)]
    assert isinstance(ws.get("reader"), torch.cuda.Event)
    assert m.data_ptr() != ws["out"].data_ptr() and mo.data_ptr() != ws["match_offsets"].data_ptr()
    want = [r for rows in oracle_rows(pats, hays, MatchKind.Standard, False) for r in rows]
    ac.count_matches_batch(hays)            # host forms reuse slot 0 on another path: the copies stay intact
    ac.find_matches_as_indexes_batch(hays)
    assert total == len(want) and [tuple(r[1:]) for r in m.tolist()] == want


# ---------------------------------------------------------------- search parity and queries
def parity_case(seed, n_hays=48):
    rng = np.random.default_rng(seed)
    pats = [[0], [5], [(1 << 21) - 1], [0, 0, 0], [5, 5 + (1 << 14)], [5, 5 + (1 << 14)],   # singles, a run of 0, duplicates
            [1, 127], [1, 127, 128], [127, 128], [1, 127, 128, 5 + (1 << 7)], [128, 5]]       # nested
    pats += [[int(x) for x in rng.choice(ALPHA, int(rng.integers(2, 6)))] for _ in range(16)]
    long_pat = [int(x) for x in rng.choice(ALPHA, 210)]   # 630 bytes: spans sieve windows
    pats.append(long_pat)
    hays = []
    for i in range(n_hays):
        h = [int(x) for x in rng.choice(ALPHA[1:], int(rng.integers(0, 120)))] if i % 7 else []
        if h and i % 3 == 0:
            at = int(rng.integers(0, len(h) + 1))
            h[at:at] = pats[i % len(pats)] * 2
        hays.append(h)
    hays[1] = [0] * 9 + hays[1] + [0] * 4            # runs of id 0 at a haystack's ends
    hays[2] = hays[2][:5] + long_pat + [7] + long_pat[:100]
    hays[-1] = hays[-1] + [0] * 7                     # ... and at the buffer's end
    return pats, hays


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("shift", [0, 1], ids=["aligned", "misaligned"])   # the encode's vector path, its scalar path
def test_search_and_queries_parity(variant, search, shift):
    kind, overlapping = search
    pats, hays = parity_case(7)
    want = oracle_rows(pats, hays, kind, overlapping)
    for h, w in zip(hays, want):
        assert w == tok_brute(pats, h, kind, overlapping)
    first_want = [rows[0] if rows else None for rows in oracle_rows(pats, hays, kind, False)]
    ac = TokenAhoCorasick(pats, kind)
    t, offs = device_batch(hays, torch.int32, shift=shift)
    with forced(variant):
        m, mo, total = ac.scan_device(t, offs, overlapping)
        assert m.dtype == torch.int32 and total == sum(map(len, want))
        mo, m = mo.tolist(), m.tolist()
        got = [[tuple(r[1:]) for r in m[mo[i]:mo[i + 1]]] for i in range(len(hays))]
        assert all(r[0] == i for i in range(len(hays)) for r in m[mo[i]:mo[i + 1]])
        assert got == want
        assert ac.find_matches_as_indexes_batch(hays, overlapping) == want
        assert ac.find_matches_as_indexes(hays[2], overlapping) == want[2]

        counts = [len(w) for w in want]
        assert ac.count_matches_device(t, offs, overlapping).tolist() == counts
        assert ac.count_matches_batch(hays, overlapping) == counts
        by_pattern = np.bincount([p for w in want for p, _, _ in w], minlength=len(pats)).tolist()
        assert ac.count_matches_by_pattern_device(t, offs, overlapping).tolist() == by_pattern
        assert ac.count_matches_by_pattern_batch(hays, overlapping) == by_pattern
        ro, pids, cnt = ac.matching_patterns_device(t, offs, overlapping)
        ro, pids, cnt = ro.tolist(), pids.tolist(), cnt.tolist()
        hits = [sorted(set(p for p, _, _ in w)) for w in want]
        assert [pids[ro[i]:ro[i + 1]] for i in range(len(hays))] == hits
        assert [cnt[ro[i]:ro[i + 1]] for i in range(len(hays))] == [[sum(1 for q, _, _ in w if q == p) for p in hs] for w, hs in zip(want, hits)]
        assert ac.matching_patterns_batch(hays, overlapping) == hits

        flags = [bool(w) for w in want]
        assert ac.is_match_device(t, offs).tolist() == flags
        assert ac.is_match_batch(hays) == flags
        rows = ac.find_first_device(t, offs).tolist()
        assert [tuple(r) if r[0] >= 0 else None for r in rows] == first_want
        assert all(r == [-1, -1, -1] for r, f in zip(rows, first_want) if f is None)
        assert ac.find_first_batch(hays) == first_want
        assert ac.find_first(hays[2]) == first_want[2]


@pytest.mark.parametrize("dtype", list(DTYPES), ids=[str(d) for d in DTYPES])
@pytest.mark.parametrize("shift", [0, 3])
def test_every_id_width_gives_the_same_rows(dtype, shift):
    rng = np.random.default_rng(11)
    alpha = [a for a in ALPHA if a < 1 << 16]
    pats = [[int(x) for x in rng.choice(alpha, int(rng.integers(1, 5)))] for _ in range(20)]
    hays = [[int(x) for x in rng.choice(alpha, int(rng.integers(0, 200)))] for _ in range(30)]
    want = oracle_rows(pats, hays, MatchKind.LeftmostLongest, False)
    ac = TokenAhoCorasick(pats, MatchKind.LeftmostLongest)
    t, offs = device_batch(hays, dtype, shift)
    m, mo, _ = ac.scan_device(t, offs)
    mo, m = mo.tolist(), m.tolist()
    assert [[tuple(r[1:]) for r in m[mo[i]:mo[i + 1]]] for i in range(len(hays))] == want
    host = [np.asarray(h, dtype=np.uint16) for h in hays]   # numpy uint16 haystacks on the host forms
    assert ac.find_matches_as_indexes_batch(host) == want


def test_issue_examples():
    assert TokenAhoCorasick([[464, 3290], [17]]).find_matches_as_indexes([9, 464, 3290, 17]) == [(0, 1, 3), (1, 3, 4)]
    assert TokenAhoCorasick([[1]]).find_matches_as_indexes([256, 0]) == []
    assert TokenAhoCorasick([[1, 2]]).find_matches_as_indexes([0, 1, 2, 1, 2]) == [(0, 1, 3), (0, 3, 5)]


def test_uint16_memmap_haystacks(tmp_path):
    rng = np.random.default_rng(3)
    ids = rng.integers(0, 50, 5000).astype(np.uint16)
    ids[100:103] = [7, 8, 9]
    path = tmp_path / "tokens.bin"
    ids.tofile(path)
    mm = np.memmap(path, dtype=np.uint16, mode="r")
    ac = TokenAhoCorasick([[7, 8, 9], [1, 2]])
    docs = [mm[0:2000], mm[2000:5000]]
    want = oracle_rows([[7, 8, 9], [1, 2]], [d.tolist() for d in docs], MatchKind.Standard, False)
    assert ac.find_matches_as_indexes_batch(docs) == want
    assert (0, 100, 103) in want[0]


# ---------------------------------------------------------------- above WINDOW_BYTES: the runs path
def test_batch_above_window_bytes_in_runs():
    ac = TokenAhoCorasick([[11, 12, 13], [12, 13], [13, 0, 13, 0]])
    limit = ac._ac.WINDOW_BYTES
    n_hays = 1000
    per = limit // 3 // n_hays + 64          # 3 x tokens > WINDOW_BYTES
    n = per * n_hays
    assert 3 * n > limit
    t = torch.full((n,), 7, dtype=torch.int32, device="cuda")   # 7 occurs in no pattern: every match lies in a plant
    offs = torch.arange(n_hays + 1, dtype=torch.int64, device="cuda") * per
    rng = np.random.default_rng(5)
    plant_sets = [[11, 12, 13], [13, 0, 13, 0, 13, 0], [12, 13, 11, 12, 13]]
    plants = []   # (haystack, token offset inside it, ids)
    for h in range(0, n_hays, 3):
        for at in (0, per - 6, int(rng.integers(10, per - 20))):   # haystack starts and ends, and one inside
            ids = plant_sets[(h + at) % 3]
            plants.append((h, at, ids))
            t[h * per + at:h * per + at + len(ids)] = torch.tensor(ids, dtype=torch.int32, device="cuda")
    for overlapping in (False, True):
        want = [[] for _ in range(n_hays)]
        for h, at, ids in plants:
            region = [7] + ids + [7]
            for p, s, e in oracle_rows(ac_pats(), [region], MatchKind.Standard, overlapping)[0]:
                want[h].append((p, at + s - 1, at + e - 1))
        want = [sorted(w, key=lambda r: (r[2], r[1], r[0])) if overlapping else sorted(w, key=lambda r: r[1]) for w in want]
        m, mo, total = ac.scan_device(t, offs, overlapping)
        assert m.dtype == torch.int64 and total == sum(map(len, want))
        mo, m = mo.tolist(), m.tolist()
        assert [[tuple(r[1:]) for r in m[mo[i]:mo[i + 1]]] for i in range(n_hays)] == want
        assert ac.count_matches_device(t, offs, overlapping).tolist() == [len(w) for w in want]
    del t
    torch.cuda.empty_cache()


def ac_pats():
    return [[11, 12, 13], [12, 13], [13, 0, 13, 0]]


# ---------------------------------------------------------------- streams
def stream_schedule(rng, n_slots, n_per_slot, alpha, pats):
    """Per slot, a queue of streams (token lists, some with patterns planted), and the feeds: (slot chunks, last flags).
    Chunks are cut at random points, with empty and one-token chunks."""
    queues = []
    for _ in range(n_slots):
        q = []
        for _ in range(n_per_slot):
            s = [int(x) for x in rng.choice(alpha, int(rng.integers(0, 80)))]
            if s and rng.random() < 0.7:
                at = int(rng.integers(0, len(s) + 1))
                s[at:at] = pats[int(rng.integers(0, len(pats)))]
            q.append(s)
        queues.append(q)
    pos = [[0, 0] for _ in range(n_slots)]   # (stream index, tokens fed)
    feeds = []
    while any(p[0] < n_per_slot for p in pos):
        chunks, lasts = [], []
        for i, (k, f) in enumerate(pos):
            if k >= n_per_slot:
                chunks.append([])
                lasts.append(False)
                continue
            s = queues[i][k]
            r = rng.random()
            size = 0 if r < 0.15 else 1 if r < 0.35 else int(rng.integers(1, 30))
            c = s[f:f + size]
            last = f + len(c) >= len(s) and rng.random() < 0.6
            chunks.append(c)
            lasts.append(last)
            pos[i] = [k + 1, 0] if last else [k, f + len(c)]
        feeds.append((chunks, lasts))
    return queues, feeds


def feed_tensors(chunks, lasts, dtype=torch.int32):
    t, offs = device_batch(chunks, dtype)
    return t, offs, torch.tensor(lasts, dtype=torch.bool, device="cuda")


STREAM_PATS = [[1, 127], [1, 127, 128, 5], [127, 128], [0, 0], [5 + (1 << 14)], [128, 5, 5 + (1 << 7), 1, 127, 128, 0]]


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_stream_batch_equals_the_stream_model(search):
    kind, overlapping = search
    rng = np.random.default_rng(21)
    ac = TokenAhoCorasick(STREAM_PATS, kind)
    orc = Oracle([enc(p) for p in STREAM_PATS], kind.name)
    max_len = ac.max_pattern_len
    queues, feeds = stream_schedule(rng, 7, 3, ALPHA, STREAM_PATS)
    sb = ac.stream_batch(7, overlapping)
    cur = [[0, 0] for _ in range(7)]   # stream index, tokens fed
    released = [0] * 7
    for chunks, lasts in feeds:
        t, offs, last = feed_tensors(chunks, lasts)
        rows, ro = sb.feed_device(t, offs, last)
        rows, ro = rows.tolist(), ro.tolist()
        for i in range(7):
            k, f = cur[i]
            if k >= 3:
                assert ro[i] == ro[i + 1]
                continue
            f += len(chunks[i])
            full = orc.find(enc(queues[i][k]), overlapping=overlapping)
            now = released_by(full, 3 * f, kind.value, overlapping, max_len, lasts[i])
            want = [(p, s // 3, e // 3) for p, s, e in now[released[i]:]]
            assert [tuple(r[1:]) for r in rows[ro[i]:ro[i + 1]]] == want
            assert all(r[0] == i for r in rows[ro[i]:ro[i + 1]])
            released[i] = len(now)
            cur[i] = [k + 1, 0] if lasts[i] else [k, f]
            if lasts[i]:
                released[i] = 0


QUERIES = [("is_match", k, False) for k in (MatchKind.Standard, MatchKind.LeftmostLongest)] + \
          [("find_first", k, False) for k in (MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest)] + \
          [("count", k, False) for k in (MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest)] + \
          [("count", MatchKind.Standard, True)]


def query_batch(ac, query, n, overlapping):
    if query == "is_match":
        return ac.is_match_stream_batch(n)
    if query == "find_first":
        return ac.find_first_stream_batch(n)
    return ac.count_matches_stream_batch(n, overlapping)


def token_answer(query, ans):
    if query == "find_first" and ans is not None:
        return (ans[0], ans[1] // 3, ans[2] // 3)
    return ans


@pytest.mark.parametrize("query,kind,overlapping", QUERIES, ids=[f"{q}-{k.name}{'-ov' if o else ''}" for q, k, o in QUERIES])
def test_query_stream_batch_equals_the_query_model(query, kind, overlapping):
    rng = np.random.default_rng(23)
    ac = TokenAhoCorasick(STREAM_PATS, kind)
    orc_kind = Oracle([enc(p) for p in STREAM_PATS], kind.name)
    orc_over = Oracle([enc(p) for p in STREAM_PATS], "Standard")
    queues, feeds = stream_schedule(rng, 6, 3, ALPHA, STREAM_PATS)
    qb = query_batch(ac, query, 6, overlapping)
    cur = [[0, 0] for _ in range(6)]
    for chunks, lasts in feeds:
        t, offs, last = feed_tensors(chunks, lasts, torch.int64)
        out = qb.feed_device(t, offs, last).tolist()
        for i in range(6):
            k, f = cur[i]
            if k >= 3:
                continue
            f += len(chunks[i])
            s = queues[i][k]
            want = token_answer(query, expected(orc_kind, orc_over, enc(s[:f]), enc(s), kind.value, ac.max_pattern_len, query,
                                                overlapping, lasts[i]))
            got = out[i]
            if query == "is_match":
                got = bool(got)
            elif query == "find_first":
                got = tuple(got) if got[0] >= 0 else None
            assert got == want, (i, k, f)
            cur[i] = [k + 1, 0] if lasts[i] else [k, f]


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_single_streams_from_the_host(search):
    kind, overlapping = search
    rng = np.random.default_rng(29)
    ac = TokenAhoCorasick(STREAM_PATS, kind)
    orc_kind = Oracle([enc(p) for p in STREAM_PATS], kind.name)
    orc_over = Oracle([enc(p) for p in STREAM_PATS], "Standard")
    s = [int(x) for x in rng.choice(ALPHA, 200)]
    s[50:50] = STREAM_PATS[1]
    s[150:150] = STREAM_PATS[5]
    cuts = sorted(int(x) for x in rng.integers(0, len(s) + 1, 12))
    chunks = [s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])]
    rows_stream = ac.stream(overlapping)
    got = [r for c in chunks for r in rows_stream.feed(np.asarray(c, dtype=np.int32))] + rows_stream.finish()
    assert got == ac.find_matches_as_indexes(s, overlapping)
    streams = {"count": ac.count_matches_stream(overlapping)}
    if not overlapping:
        streams.update(is_match=ac.is_match_stream(), find_first=ac.find_first_stream())
    for query, st in streams.items():
        f = 0
        for c in chunks:
            f += len(c)
            want = expected(orc_kind, orc_over, enc(s[:f]), enc(s), kind.value, ac.max_pattern_len, query, overlapping)
            assert st.feed(c) == token_answer(query, want)
        want = expected(orc_kind, orc_over, enc(s), enc(s), kind.value, ac.max_pattern_len, query, overlapping, True)
        assert st.finish() == token_answer(query, want)


def test_stop_sequences_one_token_per_step():
    """find_first_stream_batch of 256 generation streams fed one token per step, with stop sequences."""
    rng = np.random.default_rng(31)
    stops = [[13], [198, 198], [50256], [2, 3, 4, 5]]
    ac = TokenAhoCorasick(stops, MatchKind.LeftmostLongest)
    orc_kind = Oracle([enc(p) for p in stops], "LeftmostLongest")
    orc_over = Oracle([enc(p) for p in stops], "Standard")
    n, steps = 256, 48
    seqs = rng.integers(100, 60000, (n, steps))
    for i in range(0, n, 3):
        at = int(rng.integers(0, steps - 4))
        stop = stops[i % len(stops)]
        seqs[i, at:at + len(stop)] = stop
    fb = ac.find_first_stream_batch(n)
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda")
    done = [None] * n
    for step in range(steps):
        last = torch.full((n,), step == steps - 1, dtype=torch.bool, device="cuda")
        out = fb.feed_device(torch.from_numpy(seqs[:, step].copy()).cuda(), offs, last).tolist()
        for i in range(0, n, 5):
            s = seqs[i].tolist()
            want = token_answer("find_first", expected(orc_kind, orc_over, enc(s[:step + 1]), enc(s), 2, ac.max_pattern_len,
                                                       "find_first", False, step == steps - 1))
            got = tuple(out[i]) if out[i][0] >= 0 else None
            assert got == want, (i, step)
        for i in range(n):
            if out[i][0] >= 0 and done[i] is None:
                done[i] = tuple(out[i])
    assert sum(d is not None for d in done) >= n // 3


def test_feed_limit_is_stated_in_tokens(monkeypatch):
    from ahocorasick_rs_b200 import matcher
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 3000)
    ac = TokenAhoCorasick([[1, 2]])
    sb = ac.stream_batch(1)
    with pytest.raises(ValueError, match="at most 1000 tokens"):
        sb.feed_device(torch.zeros(1001, dtype=torch.int32, device="cuda"), torch.tensor([0, 1001], device="cuda"))
    rows, _ = sb.feed_device(torch.tensor([1, 2] * 500, dtype=torch.int32, device="cuda"), torch.tensor([0, 1000], device="cuda"))
    assert rows.shape[0] == 500
    with pytest.raises(ValueError, match="at most 1000 tokens"):
        ac.stream().feed([0] * 1001)


# ---------------------------------------------------------------- threads
def test_two_threads_share_one_object():
    pats, hays = parity_case(41, n_hays=200)
    ac = TokenAhoCorasick(pats)
    t, offs = device_batch(hays)

    def work():
        m, mo, total = ac.scan_device(t, offs, True)
        return (m.cpu().tolist(), mo.cpu().tolist(), total, ac.count_matches_device(t, offs).cpu().tolist(),
                ac.find_first_device(t, offs).cpu().tolist(), ac.find_matches_as_indexes_batch(hays[:50]))

    serial = work()
    results, errors = [], []

    def loop():
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(10):
                    results.append(work())
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)

    threads = [threading.Thread(target=loop) for _ in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert len(results) == 20 and all(r == serial for r in results)
