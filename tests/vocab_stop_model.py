"""Vocabulary stop strings without a GPU: two independent statements of each row's stop.

1. ``brute_stop``: the contract over the oracle.  Decode the row, each break starting a fresh text; run a Standard
   overlapping search over each break-free text; keep the occurrences of admitted patterns whose last byte lies in a
   new id's bytes; the stop is the one with the earliest last byte, then the longest, then the lowest pid.
2. ``StopImage``: an interpreter of acb_vocab_write's bytes that does what vocab_stop_kernel does (csrc/vocab.cuh): the
   backwards tail decode from the first new id and the walk from the root over it (VocabImage.state), then the walk over
   the new ids that stops at the first state with an admitted output and takes the first admitted pid of its list."""
import struct

from oracle import Oracle

from .vocab_model import MASK, ROOT, VocabImage


def first_new(history, new):
    """f: the row index of the first new id (new clamped to [0, len(history)])."""
    return len(history) - min(max(int(new), 0), len(history))


class BruteStop:
    """brute_stop with the oracle built once (all patterns, kind Standard)."""

    def __init__(self, patterns, vocab):
        self.vocab = [bytes(v) for v in vocab]
        self.patterns = [bytes(p) for p in patterns]
        self.orc = Oracle(self.patterns, "Standard") if patterns else None

    def __call__(self, history, new=1, admitted=None):
        """-> (pattern, token, end, length) or None."""
        if self.orc is None:
            return None
        hist = [int(c) for c in history]
        f = first_new(hist, new)
        texts, cur = [], (b"", [])   # per break-free text: its bytes and (id index, byte of the id) of each byte
        for i, c in enumerate(hist):
            if not 0 <= c < len(self.vocab):
                texts.append(cur)
                cur = (b"", [])
                continue
            v = self.vocab[c]
            cur = (cur[0] + v, cur[1] + [(i, j) for j in range(len(v))])
        texts.append(cur)
        best = None
        for text, where in texts:
            for p, s, e in self.orc.find(text, overlapping=True):
                if admitted is not None and p not in admitted:
                    continue
                i, j = where[e - 1]
                if i < f:
                    continue
                key = (i, j, -(e - s), p)
                if best is None or key < best[0]:
                    best = (key, (p, i, j + 1, e - s))
        return None if best is None else best[1]


def brute_stop(patterns, vocab, history, new=1, admitted=None):
    return BruteStop(patterns, vocab)(history, new, admitted)


class StopImage(VocabImage):
    """VocabImage with the embedded DFA's pattern lengths (ImageHeader.off_pat_len at off_dfa) and the stop walk."""

    def __init__(self, buf: bytes):
        super().__init__(buf)
        n_patterns = struct.unpack_from("<I", buf, self.off_dfa + 28)[0]
        off_pat_len = struct.unpack_from("<Q", buf, self.off_dfa + 48 + 4 * 8)[0]
        self.pat_len = struct.unpack_from(f"<{n_patterns}I", buf, self.off_dfa + off_pat_len)

    def stop(self, history, new=1, admitted=None):
        hist = [int(c) for c in history]
        f = first_new(hist, new)
        s = self.state(hist[:f])   # vocab_tail and vocab_walk over the ids before the first new one
        for i in range(f, len(hist)):
            if not 0 <= hist[i] < self.n_vocab:
                s = ROOT
                continue
            for j, b in enumerate(self.entry(hist[i])):
                e = self.step(s, b)
                s = e & MASK
                if self.hit(e, admitted):
                    pids = [int(p) for p in self.match_pid[self.match_off[s]:self.match_off[s + 1]]]
                    pid = next(p for p in pids if admitted is None or p in admitted)
                    return (pid, i, j + 1, int(self.pat_len[pid]))
        return None
