"""Float64 numpy reference of the finished-hypothesis set of beam search (b200_beam_hypotheses_update / _finalize), restated
from the Hugging Face BeamHypotheses / TensorRT-LLM convention, the reader of the kernels' state layout, and the pass rule of
the kernels against the reference (the one of beam_oracle.check_beam: scores within 1e-5 * (1 + |s|), membership and order
exact wherever the neighbouring scores are clear of that bound)."""
import copy

import numpy as np

from tests.beam_oracle import score_tol

FALSE, TRUE, NEVER = 0, 1, 2          # early_stopping


def hyp_score(cum, L, alpha):
    """cum / L^alpha in float64; exactly cum at alpha 0."""
    return float(cum) if alpha == 0 else float(cum) / float(L) ** float(alpha)


def _near(a, b, same=False):
    """Scores a and b within the tolerance of each other, and not computed from the same (cum, len) (same): the kernel's fp32
    arithmetic may order them either way. Scores of the same inputs have the same bits in the kernel too."""
    return not same and np.isfinite(a) and np.isfinite(b) and abs(a - b) <= score_tol(b)


def _same(cum_a, len_a, cum_b, len_b, alpha):
    """The two scores come from the same inputs (at alpha 0 the score is cum whatever the length)."""
    return float(cum_a) == float(cum_b) and (alpha == 0 or len_a == len_b)


class Hyps:
    """One request's set: up to W slots of dict(cum, score, len, order, tokens), in the kernel's slot order (a new hypothesis
    takes the next free slot, or the evicted one's). `ambiguous` is set once a decision compared two scores within the
    tolerance, where the kernel's fp32 arithmetic may decide the other way."""

    def __init__(self, W, max_len):
        self.W, self.max_len = W, max_len
        self.slots = []
        self.next_order = 0
        self.done = False
        self.ambiguous = False

    def worst(self):
        return min(h["score"] for h in self.slots)

    def _slot(self, s, cum, L, alpha):
        if len(self.slots) < self.W:
            return len(self.slots)
        w = min(range(self.W), key=lambda k: (self.slots[k]["score"], self.slots[k]["order"]))
        h = self.slots[w]
        self.ambiguous |= _near(s, h["score"], _same(cum, L, h["cum"], h["len"], alpha))
        return w if s > h["score"] else -1

    def add(self, cum, tokens, alpha):
        """Insert the hypothesis (cum, tokens) by the rule; True when it entered."""
        tokens = [int(t) for t in tokens]
        s = hyp_score(cum, len(tokens), alpha)
        k = self._slot(s, cum, len(tokens), alpha)
        if k < 0:
            return False
        h = dict(cum=float(cum), score=s, len=len(tokens), order=self.next_order, tokens=tokens[:self.max_len])
        self.next_order += 1
        if k == len(self.slots):
            self.slots.append(h)
        else:
            self.slots[k] = h
        return True

    def is_done(self, best, L, alpha, mode):
        """The done test on a full set: early_stopping True, else worst >= best / L^alpha (max_len^alpha for "never" at
        alpha > 0)."""
        if len(self.slots) < self.W:
            return False
        if mode == TRUE:
            return True
        if mode == NEVER and alpha > 0:
            L = self.max_len
        bound = hyp_score(best, L, alpha)
        w = min(self.slots, key=lambda h: h["score"])
        self.ambiguous |= _near(w["score"], bound, _same(w["cum"], w["len"], best, L, alpha))
        return w["score"] >= bound

    def update(self, cand_token, cand_parent, cand_score, paths, eos, alpha, mode):
        """One update from the ranked candidates [2W] of the request; paths[i]: the generated tokens of its beam i before the
        fork. A done request is left alone."""
        if self.done:
            return
        for r in range(self.W):
            c = float(cand_score[r])
            if int(cand_token[r]) != eos or not np.isfinite(c):
                continue
            self.add(c, list(paths[int(cand_parent[r])]) + [eos], alpha)
        if self.is_done(float(cand_score[0]), len(paths[int(cand_parent[0])]) + 1, alpha, mode):
            self.done = True

    def finalize(self, n, beam_cum, paths, alpha):
        """The n best, the live beams (cum beam_cum[i], tokens paths[i]) merged in first unless done; the set is unchanged.
        Returns dict(tokens [n, max_len], len, score, cum [n]; -1 / -inf for a missing one), and ranked: (score, cum, len) of
        ranks 0..n, for the gap checks of check_finalize."""
        h = copy.deepcopy(self)
        if not self.done:
            for i in range(self.W):
                if np.isfinite(beam_cum[i]) and len(paths[i]) >= 1:
                    h.add(float(beam_cum[i]), paths[i], alpha)
        ranked = sorted(h.slots, key=lambda x: (-x["score"], x["order"]))
        rk = [(x["score"], x["cum"], x["len"]) for x in ranked[:n + 1]]
        out = dict(tokens=np.full((n, self.max_len), -1, np.int64), len=np.full(n, -1, np.int64), score=np.full(n, -np.inf),
                   cum=np.full(n, -np.inf), alpha=alpha, ranked=rk + [(-np.inf, None, None)] * (n + 1 - len(rk)))
        for j, x in enumerate(ranked[:n]):
            out["tokens"][j, :len(x["tokens"])] = x["tokens"]
            out["len"][j], out["score"][j], out["cum"][j] = x["len"], x["score"], x["cum"]
        return out


def parse_state(state, B, W, max_len):
    """The kernels' state bytes (include/b200_decode_ops.h) -> per request dict(count, next_order, slots as in Hyps)."""
    raw = np.asarray(state, np.uint8)
    stride = 16 + 16 * W + 4 * W * max_len
    out = []
    for b in range(B):
        s = raw[b * stride:(b + 1) * stride]
        hd = s[:16].view(np.int32)
        meta = s[16:16 + 16 * W]
        tok = s[16 + 16 * W:].view(np.int32).reshape(W, max_len)
        f, i = meta.view(np.float32).reshape(W, 4), meta.view(np.int32).reshape(W, 4)
        slots = [dict(cum=float(f[k, 0]), score=float(f[k, 1]), len=int(i[k, 2]), order=int(i[k, 3]),
                      tokens=tok[k, :min(int(i[k, 2]), max_len)].tolist()) for k in range(int(hd[0]))]
        out.append(dict(count=int(hd[0]), next_order=int(hd[1]), slots=slots))
    return out


def check_state(got, exp, done_got, alpha, where=""):
    """One request's parsed state against the reference: slots in the same order with equal cum (bits of the fp32 candidate
    score), len, order and tokens, and scores within the tolerance; done equal. Returns True. A reference that met a near-tie
    is instead re-synchronised from the kernel's state (whose decision stands) after checking each slot's score against its
    own cum and len; returns False."""
    if exp.ambiguous:
        for h in got["slots"]:
            e = hyp_score(h["cum"], h["len"], alpha)
            assert abs(h["score"] - e) <= score_tol(e), (where, h, e)
        exp.slots = [dict(h, score=hyp_score(h["cum"], h["len"], alpha)) for h in got["slots"]]   # float64 scores again
        exp.next_order, exp.done, exp.ambiguous = got["next_order"], bool(done_got), False
        return False
    assert got["count"] == len(exp.slots), (where, got["count"], len(exp.slots))
    assert got["next_order"] == exp.next_order, (where, got["next_order"], exp.next_order)
    for k, (g, e) in enumerate(zip(got["slots"], exp.slots)):
        assert (g["len"], g["order"]) == (e["len"], e["order"]), (where, k, g, e)
        assert g["cum"] == np.float32(e["cum"]), (where, k, g["cum"], e["cum"])
        assert abs(g["score"] - e["score"]) <= score_tol(e["score"]), (where, k, g["score"], e["score"])
        assert g["tokens"] == e["tokens"], (where, k, g["tokens"], e["tokens"])
    assert bool(done_got) == exp.done, (where, done_got, exp.done)
    return True


def check_finalize(got, exp, where=""):
    """One request's finalize outputs (tokens [n, max_len], len, score, cum [n]) against Hyps.finalize: scores within the
    tolerance rank by rank (-inf where the reference has none); tokens, len and cum exact at every rank whose reference score
    is clear of its neighbours by the tolerance, or computed from the same inputs as theirs (both order those by insertion)."""
    es, rk, alpha = exp["score"], exp["ranked"], exp["alpha"]
    gs = np.asarray(got["score"], np.float64)
    n = es.shape[0]
    assert (np.isneginf(gs) == np.isneginf(es)).all(), (where, gs, es)
    fin = np.isfinite(es)
    assert (np.abs(gs[fin] - es[fin]) <= score_tol(es[fin])).all(), (where, gs, es)

    def apart(a, b):
        return not _near(a[0], b[0], a[1] is not None and b[1] is not None and _same(a[1], a[2], b[1], b[2], alpha))
    for j in range(n):
        clear = apart(rk[j], rk[j + 1]) and (j == 0 or apart(rk[j - 1], rk[j]))
        if clear:
            assert int(got["len"][j]) == exp["len"][j], (where, j, got["len"], exp["len"])
            assert np.float32(got["cum"][j]) == np.float32(exp["cum"][j]), (where, j, got["cum"], exp["cum"])
            np.testing.assert_array_equal(np.asarray(got["tokens"][j]), exp["tokens"][j], err_msg=f"{where} rank {j}")
