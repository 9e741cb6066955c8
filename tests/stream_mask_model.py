"""A Python model of the match-mask stream (acb_stream_mask_rows / acb_stream_mask_emit in include/acb200.h) on top of
tests/stream_model.py's ModelStream, and the contract it is checked against.  Per feed the model fills the two bit
spaces the device fills -- one over the seam (tail || head), one over the chunk -- from the overlapping cover of each
(overlapping) or from the rows the stream search releases (non-overlapping), then applies the release rule
R = max(0, F - halo) (R = F on `last`) and carries the held flags of [R, F)."""
from oracle import Oracle

from .stream_model import ModelStream

KIND_NAMES = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def cover(rows, n):
    """The flags of n positions covered by the spans of `rows` (pattern, start, end)."""
    bits = [0] * n
    for _, s, e in rows:
        for p in range(s, e):
            bits[p] = 1
    return bits


def one_shot_mask(pats, kind, overlapping, hay):
    """match_mask of the whole concatenation: the union of the oracle's record spans."""
    return cover(Oracle(pats, KIND_NAMES[kind]).find(hay, overlapping=overlapping), len(hay))


class MaskModelStream:
    """One stream: feed(chunk, last) -> (R_old, the flags of the bytes [R_old, R_new)).  released_positions picks the
    ones a feed at a stride returns."""

    def __init__(self, pats, kind, overlapping, over_oracle=None):
        self.rows = ModelStream(pats, kind, overlapping, over_oracle)
        self.orc = self.rows.orc
        self.overlapping = overlapping
        self.halo = self.rows.halo
        self.held = []   # the flags of [R, F)

    @property
    def released(self):
        return self.rows.fed - len(self.rows.tail)

    def feed(self, chunk: bytes, last=False):
        fed, tail = self.rows.fed, self.rows.tail
        t, head = len(tail), min(len(chunk), self.halo)
        r_old = fed - t
        assert len(self.held) == t
        if self.overlapping:
            # the cover mode on the seam and on the chunk: every match ending past F lies wholly in one of them
            seam_bits = cover(self.orc.find(tail + chunk[:head], overlapping=True), t + head)
            chunk_bits = cover(self.orc.find(chunk, overlapping=True), len(chunk))
            self.rows.feed(chunk, last)   # the advance (its rows are not used)
        else:
            seam_bits, chunk_bits = [0] * (t + head), [0] * len(chunk)
            for _, s, e in self.rows.feed(chunk, last):
                assert s >= r_old, "a released row starts before the old tail"
                for p in range(s, e):
                    if p < fed:
                        seam_bits[p - r_old] = 1
                    else:
                        chunk_bits[p - fed] = 1
        f_new = fed + len(chunk)
        r_new = f_new if last else max(0, f_new - self.halo)

        def flag(p):
            if p < fed:
                return self.held[p - r_old] | seam_bits[p - r_old]
            k = p - fed
            f = chunk_bits[k]
            if self.overlapping and k < self.halo:
                f |= seam_bits[t + k]
            return f

        out = [flag(p) for p in range(r_old, r_new)]
        self.held = [] if last else [flag(p) for p in range(r_new, f_new)]
        return r_old, out


def released_positions(r_old, flags, stride):
    """The (first index, flags) a feed returns at `stride`: the positions that are multiples of stride."""
    first = -(-r_old // stride)
    return first, flags[first * stride - r_old::stride]
