"""GPU tests (-m gpu) of the hot image's life cycle under the default engine rule (matcher._Automaton.hot,
_pick_engine, _note_trap_stats): the first profile at AUTO_PROFILE_BYTES, the re-profile after frequent traps with
its doubling back-off, the switch away from the shared-memory walker when the hot rows cover too little of the data
(to the sieve under "auto", to the segment walker that reads the tables from global memory under ENGINE = "table"),
and profiles taken from tiny and mostly empty batches.  Every call is checked against the oracle, and every
transition is read from last_stats and the per-device hot-image record."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import Implementation, MatchKind, matcher, workloads as W  # noqa: E402

from .gpu_helpers import check_batch, forced, make_ac, set_kernel  # noqa: E402

CONFIG2_PATS = [p.encode() for p in W.patterns_long()]
A_HAYS = 64            # 64 x 4 KiB haystacks: 16 384 groups, above the 4 096 a re-profile needs
RARE = b"konstantino "  # walks ten deep states of one name and matches nothing: few states, none of them in text A's profile


@pytest.fixture
def auto(monkeypatch):
    """The default engine rule, whatever ACB200_ENGINE says, with the tuning knob at auto."""
    monkeypatch.setattr(matcher._Automaton, "ENGINE", "auto")
    set_kernel(0)
    return monkeypatch


def hot_state(ac):
    return ac._ac._hot.get(torch.cuda.current_device())


def text_a(n=A_HAYS, first=0):
    _, data, offs = W.config2(n, first_index=first)
    return data, offs


def text_b(n=A_HAYS):
    line = (RARE * (4096 // len(RARE) + 1))[:4096]
    return np.frombuffer(line * n, dtype=np.uint8).copy(), np.arange(n + 1, dtype=np.int64) * 4096


def test_profile_and_reprofile_with_back_off(auto):
    ac = make_ac(CONFIG2_PATS, MatchKind.Standard, codepoints=True, implementation=Implementation.DFA)
    # 1. below AUTO_PROFILE_BYTES a fresh automaton takes the sieve and builds no hot image
    data, offs = text_a(256)
    assert data.nbytes < matcher._Automaton.AUTO_PROFILE_BYTES
    assert check_batch(CONFIG2_PATS, MatchKind.Standard, data, offs, codepoints=True, ac=ac) > 0
    assert ac._ac.last_stats["engine"] == "sieve" and ac._ac._hot == {}
    # 2. at AUTO_PROFILE_BYTES it profiles: config-2 text lives in a few hundred states
    data, offs = text_a(1100, first=256)
    assert data.nbytes >= matcher._Automaton.AUTO_PROFILE_BYTES
    assert check_batch(CONFIG2_PATS, MatchKind.Standard, data, offs, codepoints=True, ac=ac) > 0
    st = ac._ac.last_stats
    assert st["engine"] == "table" and not st["global_table"]
    assert st["hot_coverage"] >= 0.99 and st["hot_visited"] > 0
    h = hot_state(ac)
    assert h is not None and h["backoff"] == 1 and not h["reprofile"] and h["calls"] == 1
    # 3. alternate between two texts whose states lie outside each other's profile
    texts = {"A": text_a(), "B": text_b()}
    model = {"profiled": "A", "calls": 1, "backoff": 1, "reprofile": False}
    visited = st["hot_visited"]
    profiles = 0
    for name in "BBAABBBB":
        data, offs = texts[name]
        before = h
        check_batch(CONFIG2_PATS, MatchKind.Standard, data, offs, codepoints=True, ac=ac)
        st = ac._ac.last_stats
        h = hot_state(ac)
        assert st["engine"] == "table" and not st["global_table"]
        if model["reprofile"]:
            # the flag was up: this call profiled its own text, with twice the back-off
            profiles += 1
            assert h is not before and st["hot_visited"] != visited
            assert st["hot_coverage"] >= 0.99, "the inputs no longer make a well-covered profile"
            model.update(profiled=name, calls=0, backoff=2 * model["backoff"], reprofile=False)
            visited = st["hot_visited"]
        else:
            assert h is before and st["hot_visited"] == visited
        model["calls"] += 1
        frequent = st["groups"] > 4096 and st["traps"] * 10 > st["groups"]
        assert frequent == (name != model["profiled"]), (name, st)
        if frequent and model["calls"] >= model["backoff"]:
            model.update(reprofile=True, calls=0)
        assert (h["reprofile"], h["calls"], h["backoff"]) == (model["reprofile"], model["calls"], model["backoff"]), (name, h)
    assert profiles == 3 and model["backoff"] == 8


@pytest.mark.parametrize("kind,codepoints", [(MatchKind.Standard, False), (MatchKind.LeftmostLongest, False),
                                             (MatchKind.Standard, True)], ids=["Standard", "LeftmostLongest", "codepoints"])
def test_low_coverage_goes_to_the_sieve_or_the_global_table(kind, codepoints, auto):
    """A dense pattern set on random a-z: the hot rows cover too little.  "auto" answers with the sieve; ENGINE =
    "table" with the segment walker that reads the tables from global memory (kernel 4)."""
    pats, data, offs = W.config5(n_patterns=20_000, n_haystacks=1100, hay_bytes=4096)
    assert data.nbytes >= matcher._Automaton.AUTO_PROFILE_BYTES
    ac = make_ac(pats, kind, codepoints)
    assert check_batch(pats, kind, data, offs, codepoints=codepoints, ac=ac) > 500
    st = ac._ac.last_stats
    h = hot_state(ac)
    assert st["engine"] == "sieve"
    assert h is not None and h["coverage"] < 0.99 and h["rows"].reserved & 1
    auto.setattr(matcher._Automaton, "ENGINE", "table")
    assert check_batch(pats, kind, data, offs, codepoints=codepoints, ac=ac) > 500
    st = ac._ac.last_stats
    assert st["engine"] == "table" and st["global_table"] and st["hot_coverage"] < 0.99
    assert st["groups"] == 0 and st["traps"] == 0   # the staged walker counts groups; kernel 4 does not
    assert hot_state(ac) is h and not h["reprofile"]


TINY_VARIANTS = ["staged", "staged-byte-table", "staged-two-per-lane", "global-segments", "plain"]


@pytest.mark.parametrize("variant", TINY_VARIANTS)
def test_profiles_of_tiny_and_empty_batches(variant, auto):
    """A hot image profiled from a batch below 1 KiB, from a batch that is mostly empty haystacks, and built without a
    profile from an all-empty batch: those calls and the larger ones after them are correct."""
    pats = [b"he", b"she", b"his", b"hers", b"ushe", b"s", b"~x"]
    rng = np.random.default_rng(3)
    al = np.frombuffer(b"hersiux~ ", dtype=np.uint8)

    def batch(lens):
        offs = np.zeros(len(lens) + 1, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        return al[rng.integers(0, len(al), size=int(offs[-1]))].copy(), offs

    tiny = batch([40, 0, 300, 7, 1, 200])
    mostly_empty = batch([0] * 150 + [33] + [0] * 100 + [5, 0, 0, 90] + [0] * 50)
    empty = batch([0] * 20)
    big = batch(rng.integers(0, 3000, size=60).tolist())
    assert tiny[1][-1] < 1024 and mostly_empty[1][-1] < 1024 and empty[1][-1] == 0
    with forced(variant):
        for first in (tiny, mostly_empty, empty):
            for kind in (MatchKind.Standard, MatchKind.LeftmostFirst):
                ac = make_ac(pats, kind)
                for i, (data, offs) in enumerate((first, big, first)):
                    for overlapping in ((False, True) if kind == MatchKind.Standard else (False,)):
                        check_batch(pats, kind, data, offs, overlapping, ac=ac)
                        st, h = ac._ac.last_stats, hot_state(ac)
                        assert st["engine"] == "table" and h["rows"].rows == ac._ac.num_states - 1   # every state is hot
                        if i == 0 and not overlapping:
                            # a profile of the first batch's bytes leaves no re-profile pending; an image built from
                            # no bytes asks for one, and the next call with bytes takes it
                            assert (h["reprofile"], h["backoff"]) == ((True, 1) if first is empty else (False, 1))
                            assert st["hot_visited"] >= 1
                        if i == 1 and first is empty and not overlapping:
                            assert h["backoff"] == 2 and h["coverage"] >= 0.99
