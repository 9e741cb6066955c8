"""A Python model of the stream search (acb_stream_seams / acb_stream_resolve in include/acb200.h) and the contract it is
checked against.  The model takes every overlapping list from the CPU oracle's Standard automaton (the overlapping list
does not depend on the match kind), as the device takes them from the sieve, and applies what the kernels do: the
seam of each feed (tail || head), the sequence a stream selects from (every seam record, then the chunk's records that
end past the head), the selection continued from the carried restart point, and the release rule."""
import bisect

from oracle import Oracle

KIND_NAMES = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def next_selected(seq, ends, s, max_len, kind):
    """NEXT(s) over seq sorted by (end, start, pattern): the index of the record the reference's non-overlapping search
    reports once it restarts at s, or None (next_selected in csrc/capi.cu)."""
    lo = bisect.bisect_right(ends, s)
    if kind == 0:
        for j in range(lo, len(seq)):
            if seq[j][1] >= s:
                return j
        return None
    best = None
    for j in range(lo, len(seq)):
        p, st, en = seq[j]
        if best is not None and en > seq[best][1] + max_len:
            break
        if st < s:
            continue
        if best is None or st < seq[best][1]:
            best = j
        elif st == seq[best][1]:
            bp, _, be = seq[best]
            if (kind == 2 and (en > be or (en == be and p < bp))) or (kind == 1 and p < bp):
                best = j
    return best


class ModelStream:
    """One stream: feed(chunk, last) -> the rows (pattern, start, end), in bytes, that the feed releases."""

    def __init__(self, pats, kind, overlapping, over_oracle=None):
        self.orc = over_oracle or Oracle(pats, "Standard")
        self.kind = kind
        self.overlapping = overlapping
        self.max_len = max(len(p) for p in pats)
        self.halo = self.max_len - 1
        self.reset()

    def reset(self):
        self.fed, self.restart, self.tail = 0, 0, b""

    def feed(self, chunk: bytes, last=False):
        t, head = len(self.tail), min(len(chunk), self.halo)
        seam = self.tail + chunk[:head]
        seam_rows = self.orc.find(seam, overlapping=True)
        if self.overlapping:
            seam_rows = [r for r in seam_rows if r[2] > t]
        base = self.fed - t
        seq = [(p, s + base, e + base) for p, s, e in seam_rows]
        seq += [(p, s + self.fed, e + self.fed) for p, s, e in self.orc.find(chunk, overlapping=True) if e > head]
        fed_after = self.fed + len(chunk)
        if self.overlapping:
            out = seq
        else:
            ends = [r[2] for r in seq]
            out, s = [], self.restart
            while True:
                j = next_selected(seq, ends, s, self.max_len, self.kind)
                if j is None:
                    break
                if self.kind != 0 and not last and seq[j][1] + self.max_len > fed_after:
                    break
                out.append(seq[j])
                s = seq[j][2]
            self.restart = s
        self.fed = fed_after
        self.tail = (self.tail + chunk)[len(self.tail) + len(chunk) - min(fed_after, self.halo):] if self.halo else b""
        if last:
            self.reset()
        return out


def released_by(full, fed, kind, overlapping, max_len, last=False):
    """The rows of the one-shot result `full` that the release rule allows after `fed` bytes."""
    if last:
        return list(full)
    if kind == 0 or overlapping:
        return [r for r in full if r[2] <= fed]
    return [r for r in full if r[1] + max_len <= fed]
