"""Per-pattern biases for completing tokens without a GPU: the brute-force statement of the contract, and an interpreter
of the completions image (csrc/completions.h) that runs the bias kernel's algorithm (completions_bias_kernel in
csrc/completions.cuh).

For row history C and id t, P_t is the admitted pids p that t completes (p[:-1] is a suffix of C, p[-1] == t),
ordered longest pattern first, ties by ascending pid.  s = bias[p1], then s = fl32(s + bias[pj]); the logit becomes
round_L(fl32(float(logit) + s)), nearest-even, once."""
import numpy as np
import torch

from .completions_model import NONE, ComplImage

F32 = np.float32
_ieee = np.errstate(over="ignore", invalid="ignore")   # inf and NaN are part of the contract


@_ieee
def model_bias_sums(patterns, history, bias, admitted=None):
    """The statement: every admitted pattern whose p[:-1] is a suffix of the history, grouped by p[-1], each group
    summed in the contract's order in float32.  -> {t: np.float32 s}."""
    hist = [int(x) for x in history]
    terms = {}
    for pid, p in enumerate(patterns):
        if admitted is not None and pid not in admitted:
            continue
        head = [int(x) for x in p[:-1]]
        if len(head) <= len(hist) and hist[len(hist) - len(head):] == head:
            terms.setdefault(int(p[-1]), []).append((-len(p), pid))
    out = {}
    for t, ts in terms.items():
        ts.sort()
        s = F32(bias[ts[0][1]])
        for _, pid in ts[1:]:
            s = F32(s + F32(bias[pid]))
        out[t] = s
    return out


class BiasModel:
    """model_bias_sums with the patterns indexed by p[:-1] once, for many histories."""

    def __init__(self, patterns):
        self.by_head = {}
        self.K = 0
        for pid, p in enumerate(patterns):
            self.K = max(self.K, len(p))
            self.by_head.setdefault(tuple(int(x) for x in p[:-1]), []).append((pid, int(p[-1])))

    @_ieee
    def __call__(self, history, bias, admitted=None):
        hist = [int(x) for x in history]
        terms = {}
        for d in range(min(len(hist), self.K - 1), -1, -1) if self.K else ():   # longest first
            for pid, t in self.by_head.get(tuple(hist[len(hist) - d:]), ()):
                if admitted is None or pid in admitted:
                    terms.setdefault(t, []).append(pid)   # pids ascend within one length
        out = {}
        for t, pids in terms.items():
            s = F32(bias[pids[0]])
            for pid in pids[1:]:
                s = F32(s + F32(bias[pid]))
            out[t] = s
        return out


@_ieee
def apply_sums(logits, sums):
    """The expected logits: a CPU copy of `logits` (n, V) with row i's ids t of sums[i] set to
    round_L(fl32(float(logits[i, t]) + s)); every other element is copied bit for bit."""
    out = logits.detach().cpu().clone()
    rows, cols, vals = [], [], []
    f32 = out.float().numpy()
    for i, st in enumerate(sums):
        for t, s in st.items():
            rows.append(i)
            cols.append(t)
            vals.append(F32(F32(f32[i, t]) + F32(s)))
    if rows:
        out[torch.tensor(rows), torch.tensor(cols)] = torch.from_numpy(np.asarray(vals, dtype=np.float32)).to(out.dtype)
    return out


@_ieee
def interp_bias_sums(img: ComplImage, history, bias, admitted=None):
    """The kernel's algorithm over the image bytes: walk to the deepest path node v_end touching no entries, visit the
    path's nodes with entries from v_end (or its elink) along elink; the entry that is its token's first admitted
    occurrence on the path owns the token and sums the admitted entries of t at every chain node from the top down to
    its own node (a lower-bound search each), then its own node's run from its entry on.  -> {t: np.float32 s}."""
    ok = (lambda p: True) if admitted is None else (lambda p: p in admitted)
    nodes, entries = img.nodes, img.entries
    v_end = img.path(history)[-1]
    top = v_end if int(nodes[v_end, 3]) else int(nodes[v_end, 4])

    def first(v, e, t):
        fe = int(nodes[v, 2])
        k = e - 1
        while k >= fe and int(entries[k, 0]) == t:
            if ok(int(entries[k, 1])):
                return False
            k -= 1
        u = int(nodes[v, 4])
        while u != NONE:
            if any(t2 == t and ok(p2) for t2, p2 in img.node_entries(u)):
                return False
            u = int(nodes[u, 4])
        return True

    def run(k, end, t, acc):
        while k < end and int(entries[k, 0]) == t:
            pid = int(entries[k, 1])
            if ok(pid):
                acc.append(pid)
            k += 1

    out = {}
    u = top
    while u != NONE:
        fe, ne = int(nodes[u, 2]), int(nodes[u, 3])
        for e in range(fe, fe + ne):
            t, pid = int(entries[e, 0]), int(entries[e, 1])
            if not ok(pid) or not first(u, e, t):
                continue
            acc = []
            w = top
            while w != u:
                wf, wn = int(nodes[w, 2]), int(nodes[w, 3])
                lo = wf + int(np.searchsorted(entries[wf:wf + wn, 0], t, side="left"))
                run(lo, wf + wn, t, acc)
                w = int(nodes[w, 4])
            run(e, fe + ne, t, acc)
            s = F32(bias[acc[0]])
            for p in acc[1:]:
                s = F32(s + F32(bias[p]))
            assert t not in out   # one owner per id
            out[t] = s
        u = int(nodes[u, 4])
    return out
