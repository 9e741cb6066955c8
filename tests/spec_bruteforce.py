"""Declarative statement of the reference's match semantics (SURVEY.md 8c),
O(n * patterns) -- tiny inputs only.  Test infrastructure.

Let O = all occurrences (pid, a, e) with haystack[a:e] == patterns[pid]
(duplicate pattern strings are distinct pids).

* overlapping (Standard only): O sorted by (e, a, pid).
* non-overlapping: s = 0; repeat: among occurrences with a >= s take the
  minimum of  Standard (e, a, pid) | LeftmostFirst (a, pid) |
  LeftmostLongest (a, -e, pid); emit; s = e.

* pattern sets: an automaton of only the patterns in S, in their original
  relative order, with the full list's ids = the same rules over the
  occurrences of the pids in S.
"""


def occurrences(patterns, haystack):
    occ = []
    for pid, p in enumerate(patterns):
        assert len(p) > 0
        i = haystack.find(p)
        while i != -1:
            occ.append((pid, i, i + len(p)))
            i = haystack.find(p, i + 1)
    return occ


def spec_find(patterns, haystack, kind="Standard", overlapping=False, admitted=None):
    """patterns/haystack: bytes (or str, for code point semantics); admitted: a set of pids (None: all). -> [(pid, a, e)]"""
    occ = occurrences(patterns, haystack)
    if admitted is not None:
        occ = [m for m in occ if m[0] in admitted]
    if overlapping:
        if kind != "Standard":
            raise ValueError(f"match kind {kind} does not support overlapping searches")
        return sorted(occ, key=lambda m: (m[2], m[1], m[0]))
    key = {
        "Standard": lambda m: (m[2], m[1], m[0]),
        "LeftmostFirst": lambda m: (m[1], m[0]),
        "LeftmostLongest": lambda m: (m[1], -m[2], m[0]),
    }[kind]
    out, s = [], 0
    while True:
        cands = [m for m in occ if m[1] >= s]
        if not cands:
            return out
        m = min(cands, key=key)
        out.append(m)
        s = m[2]
