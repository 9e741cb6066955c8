"""A Python model of the stream queries (acb_stream_advance, acb_stream_first_resolve and acb_stream_count in
include/acb200.h): is_match, find_first and count_matches per stream after every feed, from the same seams and lists
as the stream search (tests/stream_model.py), and the answers they are checked against.  Every overlapping list comes
from the CPU oracle's Standard automaton, as the device takes them from the sieve."""
import random

from oracle import Oracle

from .stream_model import next_selected, released_by

LONG_STRETCH = 4096   # ACB_LONG_STRETCH: longer sequences are counted on the grid (patched small by the tests)


def first_order(kind, row):
    """The key order of acb_find_first, on (pattern, start, end)."""
    p, s, e = row
    return (e, s, p) if kind == 0 else (s, p) if kind == 1 else (s, -e, p)


class _Seams:
    """The carry shared by the three queries: bytes fed, tail; seam = tail || head of the chunk."""

    def __init__(self, pats, kind, over_oracle=None):
        self.orc = over_oracle or Oracle(pats, "Standard")
        self.kind = kind
        self.max_len = max(len(p) for p in pats)
        self.halo = self.max_len - 1
        self.fed, self.tail = 0, b""

    def seam(self, chunk):
        return self.tail + chunk[:min(len(chunk), self.halo)]

    def advance(self, chunk, last):
        fed_after = self.fed + len(chunk)
        self.tail = (self.tail + chunk)[len(self.tail) + len(chunk) - min(fed_after, self.halo):] if self.halo and not last else b""
        self.fed = 0 if last else fed_after


class IsMatchModel(_Seams):
    def __init__(self, pats, kind, over_oracle=None):
        super().__init__(pats, kind, over_oracle)
        self.flag = False

    def feed(self, chunk, last=False):
        # acb_any_match on the seam, then on the chunk (skipped once the flag is set)
        self.flag = self.flag or bool(self.orc.find(self.seam(chunk), overlapping=True))
        self.flag = self.flag or bool(self.orc.find(chunk, overlapping=True))
        out = self.flag
        if last:
            self.flag = False
        self.advance(chunk, last)
        return out


class FindFirstModel(_Seams):
    """state: None, ("pending", row) or ("final", row); rows in absolute bytes."""

    def __init__(self, pats, kind, over_oracle=None):
        super().__init__(pats, kind, over_oracle)
        self.state = None
        self.chunk_scans = 0

    def _best(self, rows):
        return min(rows, key=lambda r: first_order(self.kind, r)) if rows else None

    def feed(self, chunk, last=False):
        t = len(self.tail)
        if self.state is None or self.state[0] == "pending":
            cands = [self.state[1]] if self.state else []
            s = self._best(self.orc.find(self.seam(chunk), overlapping=True))
            if s is not None:
                cands.append((s[0], s[1] + self.fed - t, s[2] + self.fed - t))
            # a pending leftmost candidate starts before every record of the chunk: its scan is skipped
            if self.state is None or self.kind == 0:
                self.chunk_scans += 1
                c = self._best(self.orc.find(chunk, overlapping=True))
                if c is not None:
                    cands.append((c[0], c[1] + self.fed, c[2] + self.fed))
            best = self._best(cands)
            if best is not None:
                fed_after = self.fed + len(chunk)
                final = self.kind == 0 or last or best[1] + self.max_len <= fed_after
                self.state = ("final" if final else "pending", best)
        out = self.state[1] if self.state and self.state[0] == "final" else None
        if last:
            self.state = None
        self.advance(chunk, last)
        return out


def grid_marks(seq, head, max_len, kind, rng):
    """The chain NEXT(head), ... marked by pointer jumping (select_stretches' rule), with the order of the records inside
    each round shuffled: a mark set earlier in the same round may or may not be seen."""
    ends = [r[2] for r in seq]
    n = len(seq)
    nxt = [next_selected(seq, ends, seq[j][2], max_len, kind) for j in range(n)]
    mark = [j == head for j in range(n)]
    rounds = (n - 1).bit_length() if n > 1 else 0
    for _ in range(rounds):
        order = list(range(n))
        rng.shuffle(order)
        for j in order:
            if mark[j] and nxt[j] is not None:
                mark[nxt[j]] = True
        nxt = [nxt[nxt[j]] if nxt[j] is not None else None for j in range(n)]
    return mark


class CountModel(_Seams):
    def __init__(self, pats, kind, overlapping, over_oracle=None, seed=0):
        super().__init__(pats, kind, over_oracle)
        self.overlapping = overlapping
        self.running, self.restart = 0, 0
        self.long_stretches = 0
        self.rng = random.Random(seed)

    def feed(self, chunk, last=False):
        t = len(self.tail)
        seam_rows = self.orc.find(self.seam(chunk), overlapping=True)
        fed_after = self.fed + len(chunk)
        if self.overlapping:
            # the chunk's count (acb_count_overlapping) and the seam records across the tail / head join
            add = len(self.orc.find(chunk, overlapping=True)) + sum(1 for _, s, e in seam_rows if s < t < e)
        else:
            head = min(len(chunk), self.halo)
            base = self.fed - t
            seq = [(p, s + base, e + base) for p, s, e in seam_rows]
            seq += [(p, s + self.fed, e + self.fed) for p, s, e in self.orc.find(chunk, overlapping=True) if e > head]
            ends = [r[2] for r in seq]
            add, s = 0, self.restart
            if len(seq) <= LONG_STRETCH:
                while True:
                    j = next_selected(seq, ends, s, self.max_len, self.kind)
                    if j is None or (self.kind != 0 and not last and seq[j][1] + self.max_len > fed_after):
                        break
                    add += 1
                    s = seq[j][2]
            else:
                self.long_stretches += 1
                hd = next_selected(seq, ends, s, self.max_len, self.kind)
                if hd is not None:
                    for j, m in enumerate(grid_marks(seq, hd, self.max_len, self.kind, self.rng)):
                        if m and (self.kind == 0 or last or seq[j][1] + self.max_len <= fed_after):
                            add += 1
                            s = max(s, seq[j][2])
            self.restart = 0 if last else s
        self.running += add
        out = self.running
        if last:
            self.running = 0
        self.advance(chunk, last)
        return out


def expected(orc_kind, orc_over, prefix, final, kind, max_len, query, overlapping=False, last=False):
    """The answer after a feed: is_match(prefix); find_first(final) once the release rule allows it; the count of
    rows the stream search has released."""
    if query == "is_match":
        return bool(orc_over.find(prefix, overlapping=True))
    if query == "find_first":
        first = orc_kind.find(final, overlapping=False)[:1]
        got = released_by(first, len(prefix), kind, False, max_len, last)
        return tuple(got[0]) if got else None
    full = orc_kind.find(final, overlapping=overlapping)
    return len(released_by(full, len(prefix), kind, overlapping, max_len, last))
