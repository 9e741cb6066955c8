"""Vocabulary masks without a GPU: the image interpreter (what the kernels do) against the brute force over the oracle on
seeded vocabularies, the depth and tail_hit tables against direct computation, the C ABI's argument checks, limits and
exports, and the Python argument errors that need no device."""
import ctypes as C

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenVocabulary, _capi

from .vocab_model import (MASK, BruteModel, VocabImage, build_automaton, direct_depth, direct_tail_hit, image_bytes,
                          pack_vocab)


def _substrings(rng, text: bytes, n, lo, hi):
    out = []
    for _ in range(n):
        k = int(rng.integers(lo, hi + 1))
        a = int(rng.integers(0, max(len(text) - k, 0) + 1))
        out.append(text[a:a + k])
    return out


def _rand(rng, alpha: bytes, k):
    return np.frombuffer(alpha, dtype=np.uint8)[rng.integers(0, len(alpha), k)].tobytes()


def _case(name, rng):
    """(patterns, vocab, histories) of one seeded family."""
    alpha = b"abc"
    if name == "spanning":      # patterns of 5-9 bytes over tokens of 1-2 bytes: three or more tokens each
        pats = [_rand(rng, alpha, int(rng.integers(5, 10))) for _ in range(6)]
        vocab = [bytes([b]) for b in alpha] + _substrings(rng, b"".join(pats), 12, 1, 2)
    elif name == "long":        # a 200-byte pattern over one-byte tokens, with shorter ones beside it
        long_pat = _rand(rng, alpha, 200)
        pats = [long_pat, long_pat[50:53], b"cab"]
        vocab = [bytes([b]) for b in alpha] + [b"", long_pat[:7]]
    elif name == "mid":         # patterns inside long tokens; tokens longer than every pattern
        pats = [b"ab", b"bca", b"cc", b"abcab"]
        vocab = [bytes([b]) for b in alpha] + [_rand(rng, alpha, int(rng.integers(8, 30))) for _ in range(10)]
        vocab.append(b"xxxxxxxxxxxxabxxxxxxxxxx")
        vocab.append(b"xxxxxxxxxxxxxxxxxxxxxxxxxxx")
    elif name == "breaks":      # empty entries everywhere
        pats = [b"abc", b"ca", b"bb"]
        vocab = [b"", b"a", b"b", b"", b"c", b"ab", b"", b"bca"]
    elif name == "utf8":        # high bytes; characters split across entries
        pats = ["é".encode(), "日本".encode(), b"\xff\xfe", "aé".encode()]
        e, j = "é".encode(), "日本".encode()
        vocab = [e[:1], e[1:], j[:2], j[2:4], j[4:], b"a", b"\xff", b"\xfe\xff", "日".encode(), b"z" + e, bytes([0x80, 0xc3])]
    elif name == "nested":      # duplicates, nested patterns, one-byte patterns
        pats = [b"a", b"ab", b"ab", b"b", b"abc", b"bc", b"c"]
        vocab = [bytes([b]) for b in alpha] + [b"", b"ab", b"ca", b"x", b"xx"]
    elif name == "onebyte":     # max_pattern_len - 1 = 0: the history never matters
        pats = [b"a", b"\x00", b"a"]
        vocab = [b"a", b"b", b"\x00", b"ba", b"", b"bbb"]
    elif name == "none":        # no patterns: nothing completes
        pats = []
        vocab = [b"a", b"", b"ab"]
    else:
        raise AssertionError(name)
    n = len(vocab)
    hists = [[], [-1], [n], [n + 7, 0]]
    for i in range(24):
        h = [int(x) for x in rng.integers(0, n, int(rng.integers(0, 12 if name != "long" else 260)))]
        if name == "long" and i % 3 == 0:   # most of the long pattern, one byte per token (the one-byte entries lead)
            cut = int(rng.integers(150, 200))
            h = [alpha.index(b) for b in long_pat[:cut]]
        if i % 4 == 1 and h:   # a break at the start, in the middle or at the end
            h.insert(int(rng.integers(0, len(h) + 1)), int(rng.choice([-1, -100, n, n + 3])))
        hists.append(h)
    return pats, vocab, hists


CASES = ["spanning", "long", "mid", "breaks", "utf8", "nested", "onebyte", "none"]


def _subsets(rng, n_pats):
    return [None, set(), {p for p in range(n_pats) if rng.random() < 0.5}]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("seed", range(2))
def test_interpreter_equals_brute_force(name, seed):
    rng = np.random.default_rng(1000 * seed + CASES.index(name))
    pats, vocab, hists = _case(name, rng)
    brute = BruteModel(pats, vocab)
    images = [VocabImage(image_bytes(pats, vocab, kind)) for kind in (0, 1, 2)]
    for S in _subsets(rng, len(pats)):
        for h in hists:
            want = brute(h, S)
            for kind, img in enumerate(images):   # every match kind gives one answer
                assert img.completing(h, S) == want, (name, kind, h, S)
    # V below n_vocab: the candidates stop at V
    h = hists[-1]
    assert images[0].completing(h, None, V=2) == [t for t in brute(h) if t < 2]


def test_worked_example():
    pats = [b"damn", b"\nUser:"]
    vocab = [b"d", b"am", b"n", b"damn", b"\n", b"User", b":", b"hello"]
    img = VocabImage(image_bytes(pats, vocab))
    brute = BruteModel(pats, vocab)
    for h, want in (([0, 1], [2, 3]), ([4, 5], [3, 6]), ([4, -1, 5], [3])):
        assert img.completing(h) == want and brute(h) == want


def test_the_history_beyond_the_longest_pattern_does_not_matter():
    pats = [b"abcd"]
    vocab = [b"a", b"b", b"c", b"d", b"xab"]
    img = VocabImage(image_bytes(pats, vocab))
    assert img.need == 3
    assert img.completing([0, 1, 2]) == [3] and img.completing([4, 2]) == [3]
    assert img.completing([1, 1, 4, 2]) == [3]   # only the last three bytes, "abc", are read
    assert img.completing([4]) == [] and img.completing([0, 1]) == []


def test_utf8_character_split_across_tokens():
    ac_pats = ["é", "naïve"]
    enc = [p.encode() for p in ac_pats]
    vocab = [b"na", b"\xc3", b"\xaf", b"ve", b"\xa9"]
    img = VocabImage(image_bytes(enc, vocab))
    assert img.completing([1]) == [4]             # "\xc3" + "\xa9" = "é"
    assert img.completing([0, 1, 2]) == [3]       # "na" "\xc3" "\xaf" + "ve"
    assert BruteModel(enc, vocab)([0, 1, 2]) == [3]


# ---- the tables --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_depth_and_tail_hit_tables(name):
    rng = np.random.default_rng(7 + CASES.index(name))
    pats, vocab, _ = _case(name, rng)
    for kind in (0, 1, 2):
        img = VocabImage(image_bytes(pats, vocab, kind))
        assert img.magic == 0x31564341 and img.n_vocab == len(vocab)
        assert img.max_pat_len == max((len(p) for p in pats), default=0)
        d = direct_depth(img.trans)
        assert np.array_equal(img.depth[1:], d[1:])
        assert np.all(np.diff(img.depth[1:].astype(np.int64)) >= 0)   # breadth-first: depth never decreases
        assert img.lvl2 == next((s for s in range(1, img.n_states) if img.depth[s] >= 2), img.n_states)
        want = direct_tail_hit(pats, vocab)
        assert img.tail.tolist() == want
        assert img.n_tail_hits == sum(t >= 0 for t in want)
        for t, v in enumerate(vocab):
            assert bytes(img.entry(t)) == v
        # the DFA is a Standard one whatever the kind: a copy of the automaton's own only when it is Standard
        L, h = build_automaton(pats, 0)
        try:
            standard_bytes = int(L.acb_image_bytes(h))
        finally:
            L.acb_free(h)
        assert img.extra == (0 if kind == 0 else standard_bytes)


def test_first_byte_share_is_most_ids_on_text_like_vocabularies():
    rng = np.random.default_rng(3)
    text = b"the quick brown fox jumps over the lazy dog; " * 20
    pats = _substrings(rng, text, 40, 3, 8)
    vocab = [bytes([b]) for b in range(256)] + _substrings(rng, text, 300, 2, 6)
    img = VocabImage(image_bytes(pats, vocab))
    s_hist = [int(x) for x in rng.integers(0, len(vocab), 20)]
    assert img.first_byte_ids(s_hist) > 0.5 * sum(1 for v in vocab if v)


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_exports():
    L = _capi.lib()
    for name in ("acb_vocab_build", "acb_vocab_write", "acb_vocab_describe", "acb_vocab_mask"):
        assert name in _capi.EXPORTS and getattr(L, name)


def test_build_write_describe():
    pats = [b"ab", b"abc"]
    vocab = [b"a", b"bc", b"abc", b""]
    for kind in (0, 2):
        L, h = build_automaton(pats, kind)
        try:
            blob, offs = pack_vocab(vocab)
            n = C.c_uint64(0)
            assert L.acb_vocab_build(h, blob.ctypes.data, offs.ctypes.data, 4, C.byref(n)) == _capi.ACB_OK
            buf = np.zeros(n.value, dtype=np.uint8)
            assert L.acb_vocab_write(h, blob.ctypes.data, offs.ctypes.data, 4, buf.ctypes.data, n.value - 1) == _capi.ACB_ECAPACITY
            assert L.acb_vocab_write(h, blob.ctypes.data, offs.ctypes.data, 4, buf.ctypes.data, n.value) == _capi.ACB_OK
            d = _capi.VocabDesc()
            assert L.acb_vocab_describe(buf.ctypes.data, C.byref(d)) == _capi.ACB_OK
            assert (d.n_vocab, d.max_pattern_len, d.tail_hit_ids) == (4, 3, 1)
            assert (d.extra_dfa_bytes == 0) == (kind == 0)
            assert d.states == int(L.acb_num_states(h)) or kind != 0
            bad = np.zeros(64, dtype=np.uint8)
            assert L.acb_vocab_describe(bad.ctypes.data, C.byref(d)) == _capi.ACB_EINVAL
            assert L.acb_vocab_describe(None, C.byref(d)) == _capi.ACB_EINVAL
        finally:
            L.acb_free(h)


def test_build_argument_errors_and_limits():
    L, h = build_automaton([b"ab"])
    try:
        n = C.c_uint64(0)
        blob = np.frombuffer(b"abc", dtype=np.uint8)

        def build(offs, count, b=blob):
            o = np.asarray(offs, dtype=np.uint64)
            return L.acb_vocab_build(h, None if b is None else b.ctypes.data, o.ctypes.data, count, C.byref(n))

        assert build([0, 1, 3], 2) == _capi.ACB_OK
        assert build([1, 2, 3], 2) == _capi.ACB_EINVAL          # offsets[0] != 0
        assert build([0, 2, 1], 2) == _capi.ACB_EINVAL          # decreasing
        assert build([0, 2, 3], 2, None) == _capi.ACB_EINVAL    # bytes without a blob
        assert build([0, 0, 0], 2, None) == _capi.ACB_OK        # no bytes: no blob needed
        assert build([0], 0, None) == _capi.ACB_OK and n.value > 0
        assert L.acb_vocab_build(h, blob.ctypes.data, None, 1, C.byref(n)) == _capi.ACB_EINVAL
        assert L.acb_vocab_build(None, blob.ctypes.data, np.zeros(2, np.uint64).ctypes.data, 1, C.byref(n)) == _capi.ACB_EINVAL
        assert L.acb_vocab_build(h, blob.ctypes.data, np.zeros(2, np.uint64).ctypes.data, 1, None) == _capi.ACB_EINVAL
        # the byte limit at its edge: the build reads the offsets, not the bytes
        assert build([0, _capi.ACB_VOCAB_MAX_BYTES], 1) == _capi.ACB_OK and n.value > _capi.ACB_VOCAB_MAX_BYTES
        assert build([0, _capi.ACB_VOCAB_MAX_BYTES + 1], 1) == _capi.ACB_EINVAL
        assert "bytes" in _capi.last_error()
        # the id limit: refused before any offset past the first is read
        assert build([0], _capi.ACB_VOCAB_MAX_IDS + 1) == _capi.ACB_EINVAL
        assert "ACB_VOCAB_MAX_IDS" in _capi.last_error()
        buf = np.zeros(16, dtype=np.uint8)
        o = np.asarray([0, 1, 3], dtype=np.uint64)
        assert L.acb_vocab_write(h, blob.ctypes.data, o.ctypes.data, 2, None, 16) == _capi.ACB_EINVAL
        assert L.acb_vocab_write(h, blob.ctypes.data, o.ctypes.data, _capi.ACB_VOCAB_MAX_IDS + 1, buf.ctypes.data, 16) == _capi.ACB_EINVAL
    finally:
        L.acb_free(h)


def _mask(L, h, **kw):
    img = np.zeros(16, dtype=np.uint8)
    tok = np.zeros(4, dtype=np.int64)
    off = np.array([0, 2], dtype=np.int64)
    st = np.zeros(4, dtype=np.uint32)
    lg = np.zeros(8, dtype=np.float32)
    a = dict(a=h, img=img.ctypes.data, tok=tok.ctypes.data, tb=8, nt=4, off=off.ctypes.data, nr=1, st=st.ctypes.data, lg=lg.ctypes.data,
             dt=_capi.ACB_LOGITS_F32, rs=8, V=8, value=float("-inf"), flt=None)
    a.update(kw)
    return L.acb_vocab_mask(a["a"], a["img"], a["tok"], a["tb"], a["nt"], a["off"], a["nr"], a["st"], a["lg"], a["dt"], a["rs"], a["V"],
                            a["value"], a["flt"], None)


def test_mask_argument_errors_before_any_cuda_call():
    L, h = build_automaton([b"ab"])
    try:
        E = _capi.ACB_EINVAL
        for kw in (dict(a=None), dict(img=None), dict(tok=None), dict(off=None), dict(st=None), dict(lg=None), dict(tb=3), dict(tb=1),
                   dict(nt=1 << 60), dict(nr=-1), dict(nr=1 << 32), dict(dt=3), dict(dt=-1), dict(V=0), dict(V=1 << 62), dict(rs=-1),
                   dict(rs=1 << 62)):
            assert _mask(L, h, **kw) == E, kw
        f = _capi.PatternFilter()
        f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = None, 1, None, 4
        assert _mask(L, h, flt=C.byref(f)) == E
        bits = np.zeros(1, dtype=np.uint32)
        f.dev_set_bits, f.n_sets = bits.ctypes.data, 0
        assert _mask(L, h, flt=C.byref(f)) == E
        f.n_sets, f.index_bytes = 1, 2
        assert _mask(L, h, flt=C.byref(f)) == E
        f.n_sets, f.index_bytes, f.dev_set_index = (1 << 32) - 1, 4, bits.ctypes.data   # set indexes are 32-bit in the kernel
        assert _mask(L, h, flt=C.byref(f)) == E and "n_sets" in _capi.last_error()
    finally:
        L.acb_free(h)


# ---- Python argument errors that need no device --------------------------------------------------------------------------
def test_vocabulary_entries_must_be_bytes():
    ac = BytesAhoCorasick([b"ab"])
    with pytest.raises(TypeError, match="str"):
        ac.vocabulary([b"a", "Ġb"])
    with pytest.raises(TypeError):
        ac.vocabulary(b"abc")
    with pytest.raises(TypeError):
        ac.vocabulary("abc")
    with pytest.raises(TypeError):
        ac.vocabulary([b"a", 5])
    v = AhoCorasick(["é"]).vocabulary([b"\xc3", bytearray(b"\xa9"), memoryview(b""), np.frombuffer(b"xy", dtype=np.uint8)])
    assert isinstance(v, TokenVocabulary) and v.n_vocab == 4
    assert v.image_bytes > 0
    assert BytesAhoCorasick([b"ab"]).vocabulary([]).n_vocab == 0


def test_vocabulary_of_every_match_kind_builds():
    for kind in MatchKind:
        v = BytesAhoCorasick([b"ab", b"abc"], matchkind=kind).vocabulary([b"a", b"bc"])
        assert v.n_vocab == 2


def test_mask_argument_errors_without_a_device():
    v = BytesAhoCorasick([b"ab"]).vocabulary([b"a", b"b"])
    with pytest.raises(TypeError, match="tokens"):
        v.mask_completing_tokens_(torch.zeros(1, 2), torch.zeros(2, dtype=torch.int64), torch.tensor([0, 2]))
    with pytest.raises(TypeError, match="tokens"):
        v.mask_completing_tokens_(torch.zeros(1, 2), [0, 1], torch.tensor([0, 2]))


def test_history_errors_without_a_device():
    v = BytesAhoCorasick([b"ab"]).vocabulary([b"a", b"b"])
    with pytest.raises(TypeError):
        v.completing_tokens([[0, 1], [1]])
    with pytest.raises(TypeError):
        v.completing_tokens([0.5, 1.0])
    with pytest.raises(TypeError):
        v.completing_tokens(["a"])
    with pytest.raises(ValueError):
        v.completing_tokens_batch([[0], [1]], patterns=[[0]])


# ---- the compiled mask kernel ----------------------------------------------------------------------------------------
def test_mask_kernel_stores_use_no_uniform_row_index():
    """ptxas (CUDA 12.9) once compiled the 16-bit filtered mask kernel's store address from a uniform register (R2UR of
    the per-thread row counter) while the lanes of a warp were at different rows, sending some bans to another row of
    the tile (DESIGN §4.18).  The kernel now stores after its walks, each row from the thread's own bits; no instance may
    move a per-thread value into a uniform register after the tile barrier."""
    import os
    import shutil
    import subprocess
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed")
    out = subprocess.run([tool, "-sass", _capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    seen, fn, barrier = set(), None, False
    for line in out.splitlines():
        if "Function :" in line:
            fn, barrier = line.split("Function :")[1].strip(), False
            if "vocab_mask_kernel" in fn:
                seen.add(fn)
        elif fn and "vocab_mask_kernel" in fn:
            barrier = barrier or "BAR.SYNC" in line
            assert not (barrier and "R2UR" in line), (fn, line.strip())
    assert len(seen) == 6
