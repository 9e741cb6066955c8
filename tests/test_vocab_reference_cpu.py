"""The DFA-free vocabulary reference (tests/vocab_reference.py) against the two statements in tests/vocab_model.py,
without a GPU: the brute force over the oracle on every family of test_vocab_cpu, and the image interpreter on the
geometry families of tests/vocab_families.py (so the interpreter's backwards scan is checked at 2 to 32 history pieces
against something other than itself)."""
import numpy as np
import pytest

from . import table_shapes as ts
from . import vocab_families as vf
from .test_vocab_cpu import CASES, _case, _subsets
from .vocab_model import BruteModel, VocabImage, image_bytes
from .vocab_reference import VocabReference, tail_bytes


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("seed", range(2))
def test_reference_equals_brute_force(name, seed):
    rng = np.random.default_rng(1000 * seed + CASES.index(name))
    pats, vocab, hists = _case(name, rng)
    brute, ref = BruteModel(pats, vocab), VocabReference(pats, vocab)
    n = len(vocab)
    for S in _subsets(rng, len(pats)):
        for h in hists:
            for V in (None, n - 1, n, n + 5):
                assert ref(h, S, V) == brute(h, S, V), (name, h, S, V)


def test_tail_and_prefix_ranges():
    vocab = [b"\xff", b"\xff\xff", b"\xffa", b"", b"b", b"ab", b"\xfe\xff"]
    ref = VocabReference([b"a\xff\xff", b"x\xfe"], vocab)
    assert tail_bytes(vocab, [4, -1, 5, 3]) == b"ab" and tail_bytes(vocab, [7]) == b""
    assert sorted(ref.starting_with(b"\xff").tolist()) == [0, 1, 2]
    assert sorted(ref.starting_with(b"\xff\xff").tolist()) == [1]
    assert ref([5]) == [] and ref([3, 0, 5, 3]) == []
    assert ref([4, 2]) == [1] and ref([2, 0]) == [0, 1, 2]   # "b\xffa" + "\xff\xff"; "\xffa\xff" + "\xff.."
    assert ref([-1]) == [] and VocabReference([b"x\xfe"], vocab)([]) == []
    brute = BruteModel([b"a\xff\xff", b"x\xfe"], vocab)
    for h in ([4, 2], [2, 0], [2], [5, 0], [6, 5]):
        assert ref(h) == brute(h), h


def _families():
    out = [vf.pieces(L) for L in vf.PIECE_LENS] + [f() for f in vf.WALKS]
    return out + [vf.shape_family(c, n_hist=8) for c in ts.CASES]


FAMILIES = _families()


@pytest.mark.parametrize("fam", FAMILIES, ids=[f.name for f in FAMILIES])
def test_reference_equals_interpreter_on_geometry_families(fam):
    rng = np.random.default_rng(7)
    ref = VocabReference(fam.patterns, fam.vocab)
    subsets = [None, {p for p in range(len(fam.patterns)) if rng.random() < 0.5}, {len(fam.patterns) - 1}]
    if fam.name == "shadowed":
        subsets.append({1})
    kinds = (0, 1, 2) if fam.name in ("shadowed", "filtered-tails") or fam.name.startswith("shape-") else (0,)
    for kind in kinds:
        img = VocabImage(image_bytes(fam.patterns, fam.vocab, kind))
        assert img.need == fam.need
        hists = fam.histories if len(fam.vocab) < 2000 else fam.histories[::4]
        for S in subsets:
            for h in hists:
                assert img.completing(h, S) == ref(h, S), (fam.name, kind, S, h)


def test_pieces_reach_every_lane_and_piece_targeted():
    """The piece families stop the scan at lane 0 and lane 31 of the second and third piece, and read 32 pieces."""
    stops = set()
    for L in vf.PIECE_LENS:
        fam = vf.pieces(L)
        for h in fam.histories:
            k = vf.read_stop(fam.vocab, h, fam.need)
            stops.add((k // 32, k % 32))
    assert {(1, 0), (1, 31), (2, 0), (2, 31)} <= stops
    assert max(p for p, _ in stops) >= 31


def test_walk_families_reach_their_branches():
    img = VocabImage(image_bytes(vf.one_byte().patterns, vf.one_byte().vocab))
    assert img.lvl2 == img.n_states and img.need == 0
    deep = vf.deep_state()
    img = VocabImage(image_bytes(deep.patterns, deep.vocab))
    assert max(int(img.depth[img.state(h)]) for h in deep.histories) >= 150
    assert max(len(v) for v in deep.vocab) >= 150
    ft = vf.filtered_tails()
    img = VocabImage(image_bytes(ft.patterns, ft.vocab))
    t = ft.vocab.index(b"qqxyqq")
    assert int(img.tail[t]) == 3 and not img.banned(img.state([]), t, {1})      # tail_hit past j, no admitted hit
    t = ft.vocab.index(b"qqxyqqzw")
    assert int(img.tail[t]) == 7 and img.banned(img.state([]), t, {1})          # the admitted hit is the tail byte
    sh = vf.shadowed()
    for kind in (1, 2):
        assert VocabImage(image_bytes(sh.patterns, sh.vocab, kind)).extra > 0
