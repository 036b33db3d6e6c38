"""b200_sample (csrc/sampling.cuh) at the edges a comparison with the float64 oracle cannot resolve: the inverse-CDF draw at
its chunk boundaries, checked token for token against an exact float32 emulation of the kernel's chunk sums and block scan;
the top-k / top-p kept sets against the kernel's own probabilities; masked logits; penalties at their edges; row
independence and determinism; and the op behind an lm_head GEMM under PDL in a CUDA graph."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402

dev = torch.device("cuda")
F32 = np.float32
THREADS = 1024                                  # kSampleThreads: thread t sums tokens [t * per, (t + 1) * per)
BELOW_ONE = np.nextafter(F32(1), F32(0))        # the largest uniform the op accepts
MAX_ROWS = 2048                                 # probes per launch (one row per probe)


class Draw:
    """Exact float32 emulation of the kernel's draw for one row, built from what the kernel leaves behind: its probabilities
    p (written over the logits) and its kept set (probs_out > 0; a kept token with p == 0 adds nothing to any sum). The
    library is built without fast-math, so every fp32 add rounds to nearest and keeps subnormals, as numpy's adds do."""

    def __init__(self, p, kept):
        V = p.size
        self.p, self.kept = p, kept & (p > 0)
        self.per = -(-V // THREADS)
        vals = np.zeros(THREADS * self.per, F32)
        vals[:V] = np.where(self.kept, p, F32(0))
        self.chunks = vals.reshape(THREADS, self.per)
        mine = np.zeros(THREADS, F32)
        for j in range(self.per):                   # each chunk summed sequentially in index order
            mine = mine + self.chunks[:, j]
        s = mine.copy()
        off = 1
        while off < THREADS:                        # Hillis-Steele inclusive scan: s[t] += s[t - off], off = 1, 2, ..., 512
            s[off:] = s[off:] + s[:-off]
            off *= 2
        self.mine, self.scan, self.total = mine, s, s[-1]
        self.start = np.concatenate([np.zeros(1, F32), s[:-1]])       # chunk t starts where the prefix before it ends
        self.pos = np.flatnonzero(mine > 0)
        self._walks = {}

    def product(self, u):
        return np.asarray(u, F32) * self.total

    def target(self, u):
        """fl(u * total), clamped below total."""
        return np.minimum(self.product(u), np.nextafter(self.total, F32(0)))

    def token(self, u, argmax=False):
        """The token the kernel must return: the last chunk with mass whose start is <= target owns the target, and walks
        its kept tokens with p > 0 until the running sum passes the target (its last one if rounding never lets it)."""
        tgt = F32(0) if argmax else self.target(u)
        owner = self.pos[self.start[self.pos] <= tgt].max()
        if owner not in self._walks:
            idx = owner * self.per + np.flatnonzero(self.chunks[owner])
            run = np.add.accumulate(np.concatenate([self.start[owner:owner + 1], self.p[idx]]), dtype=F32)[1:]
            self._walks[owner] = idx, run
        idx, run = self._walks[owner]
        hit = np.flatnonzero(run > tgt)
        return int(idx[hit[0]] if hit.size else idx[-1])

    def gaps(self):
        """Target ranges [a, b) that no chunk owns when each chunk recomputes its own interval [scan - mine, scan): the
        intervals are rounded separately, so consecutive ones need not meet."""
        lo, hi = (self.scan - self.mine)[self.pos], self.scan[self.pos]
        order = np.argsort(lo, kind="stable")
        out, cur = [], F32(0)
        for a, b in zip(lo[order], hi[order]):
            if a > cur:
                out.append((cur, a))
            cur = max(cur, b)
        if cur < self.total:
            out.append((cur, self.total))
        return out

    def u_reaching(self, g):
        """For each target g: the smallest u in [0, 1) with fl(u * total) >= g, or nan when no such u exists."""
        g = np.asarray(g, F32)
        u = np.clip((g.astype(np.float64) / float(self.total)).astype(F32), F32(0), F32(1))
        for _ in range(64):
            low = self.product(u) < g
            if not low.any():
                break
            u[low] = np.nextafter(u[low], F32(2))
        for _ in range(64):
            prev = np.nextafter(u, F32(-1))
            down = (u > 0) & (self.product(prev) >= g)
            if not down.any():
                break
            u[down] = prev[down]
        assert (self.product(u) >= g).all() and ((u == 0) | (self.product(np.nextafter(u, F32(-1))) < g)).all()
        return np.where(u <= BELOW_ONE, u, np.nan).astype(F32)

    def probes(self):
        """Uniforms whose target lands on every chunk boundary and one float below it, inside every gap, at 0 and at the
        largest uniform below 1. Returns (u, number of gap probes)."""
        bounds = np.unique(np.concatenate([self.start[self.pos], (self.scan - self.mine)[self.pos], self.scan[self.pos]]))
        at = self.u_reaching(bounds)
        below = np.nextafter(at, F32(-1))
        gaps = np.array(self.gaps(), F32).reshape(-1, 2)
        gu = self.u_reaching(gaps[:, 0])
        gu = gu[~np.isnan(gu) & (self.product(np.nan_to_num(gu)) < gaps[:, 1])]      # some gaps no product can land in
        u = np.concatenate([at, below[below >= 0], gu, np.array([0, BELOW_ONE], F32)])
        return np.unique(u[~np.isnan(u)]).astype(F32), gu.size

    def cdf_interval(self, tok):
        """The token's [lo, hi) interval of the float64 CDF over the kept probabilities, in units of u."""
        q = np.where(self.kept, self.p, 0).astype(np.float64)
        c = np.cumsum(q)
        return (c[tok] - q[tok]) / c[-1], c[tok] / c[-1]

    def slack(self):
        """Rounding allowance of the draw in units of u: the chunk sum and the walk each add up to `per` terms, the scan
        adds 10 levels, plus the product u * total and the clamp; each step errs by at most one ulp of total."""
        return (2 * self.per + 12) * float(np.spacing(self.total)) / float(self.total)


def _t(a, dt):
    return None if a is None else torch.tensor(np.asarray(a), dtype=dt, device=dev)


def _sample_copies(row, u, top_k, top_p, temperature=None):
    """Run len(u) copies of one logits row, one uniform each. Returns (tokens, token_prob, p, probs_out of the row)."""
    V = row.size
    toks, tprobs, p, probs = [], [], None, None
    base = torch.from_numpy(row).to(dev)
    for s in range(0, len(u), MAX_ROWS):
        uu = u[s:s + MAX_ROWS]
        n = len(uu)
        x = base.expand(n, V).contiguous()
        tok, tprob, pr = ops.sample(x, _t([top_k] * n, torch.int32), _t([top_p] * n, torch.float32), _t(uu, torch.float32),
                                    temperature=None if temperature is None else _t([temperature] * n, torch.float32),
                                    want_probs=True)
        torch.cuda.synchronize()
        assert torch.equal(x, x[:1].expand_as(x)) and torch.equal(pr, pr[:1].expand_as(pr)), "copies of one row differ"
        if p is None:
            p, probs = x[0].cpu().numpy(), pr[0].cpu().numpy()
        else:
            assert np.array_equal(p, x[0].cpu().numpy()) and np.array_equal(probs, pr[0].cpu().numpy())
        toks.append(tok.cpu().numpy())
        tprobs.append(tprob.cpu().numpy())
    return np.concatenate(toks), np.concatenate(tprobs), p, probs


def _check_draws(u, tok, tprob, p, probs, what):
    """Every draw: a kept token with p > 0, token_prob == probs_out[token], u inside the token's float64 CDF interval up to
    the draw's rounding allowance, and exactly the token the emulation predicts."""
    d = Draw(p, probs > 0)
    lo, hi = d.cdf_interval(tok)
    sl = d.slack()
    exp = np.array([d.token(x) for x in u])
    bad_kept = ~((probs[tok] > 0) & (p[tok] > 0))
    bad_prob = tprob.view(np.uint32) != probs[tok].view(np.uint32)
    bad_cdf = ~((u >= lo - sl) & (u < hi + sl))
    bad_tok = tok != exp
    bad = bad_kept | bad_prob | bad_cdf | bad_tok
    if bad.any():
        i = np.flatnonzero(bad)
        ex = ", ".join(f"u={u[j]!r} -> {tok[j]} (p {p[tok[j]]:.3g}, emulated {exp[j]})" for j in i[:8])
        pytest.fail(f"{what}: {bad.sum()} of {u.size} draws wrong (not kept or p == 0: {bad_kept.sum()}, token_prob != "
                    f"probs_out: {bad_prob.sum()}, outside the CDF step: {bad_cdf.sum()}, not the emulated token: "
                    f"{bad_tok.sum()}; returned token 0: {(tok[i] == 0).sum()}); e.g. {ex}")
    return d


VOCABS = [1, 7, 1000, 1024, 1025, 32000, 128256, 152064, 256000]


def _filtered_row(V, filt, rng):
    """(logits, top_k, top_p, temperature) of one filter case."""
    if filt == "none":                       # everything kept: every chunk has mass
        return (rng.standard_normal(V) * 3).astype(F32), 0, 1.0, None
    if filt == "dense":                      # top-k then top-p over a flat row: most chunks keep some and drop some tokens
        return rng.standard_normal(V).astype(F32), max(V // 2, 1), 0.9, None
    if filt == "sparse":                     # top-k 50: most chunks are empty and the owners lie far apart
        return (rng.standard_normal(V) * 3).astype(F32), 50, 1.0, None
    # low temperature: most of the row underflows to p == 0 (still kept: no filter), the last third as whole chunks
    lg = (rng.standard_normal(V) * 3).astype(F32)
    lg[2 * V // 3:] -= 200
    return lg, 0, 1.0, 0.05


@pytest.mark.parametrize("filt", ["none", "dense", "sparse", "underflow"])
@pytest.mark.parametrize("V", VOCABS)
def test_draw_at_chunk_boundaries_and_gaps(V, filt):
    rng = np.random.default_rng(V * 4 + len(filt))
    lg, top_k, top_p, temp = _filtered_row(V, filt, rng)
    # a first run gives the kernel's own probabilities, from which the probes are placed
    _, _, p, probs = _sample_copies(lg, np.zeros(1, F32), top_k, top_p, temp)
    u, n_gap = Draw(p, probs > 0).probes()
    tok, tprob, p2, probs2 = _sample_copies(lg, u, top_k, top_p, temp)
    assert np.array_equal(p, p2) and np.array_equal(probs, probs2)
    _check_draws(u, tok, tprob, p, probs, f"V={V} {filt} ({n_gap} gap probes)")
    if filt == "underflow" and V >= 1000:
        assert (p == 0).mean() > 0.5, "the low-temperature row should underflow most of the vocabulary"


def _spread(V, n, per, first_chunk):
    """n token indices in distinct chunks, far apart, in descending chunk order."""
    chunks = np.linspace(first_chunk, min(THREADS - 1, (V - 1) // per), n).astype(int)[::-1]
    return np.minimum(chunks * per + (np.arange(n) % per), V - 1)


@pytest.mark.parametrize("V", [1000, 32000, 128256])
def test_top_k_keeps_exactly_the_tokens_at_or_above_the_kth_probability(V):
    rng = np.random.default_rng(V)
    per = -(-V // THREADS)
    lg = np.minimum(rng.standard_normal(V) * 2, 5).astype(F32)
    ties = _spread(V, 4, per, 3)                             # four equal logits in different chunks
    lg[ties] = 6.0
    above = rng.choice(np.setdiff1d(np.arange(V), ties), 38, replace=False)
    lg[above] = 7.0 + np.arange(38, dtype=F32) * 0.01        # 38 distinct values above the ties
    ks = [1, 2, 37, 38, 39, 40, 41, 42, 43, 100]             # 39..42 straddle the tie group
    n = len(ks)
    x = torch.from_numpy(lg).to(dev).expand(n, V).contiguous()
    u = rng.random(n).astype(F32)
    tok, tprob, probs = ops.sample(x, _t(ks, torch.int32), _t([1.0] * n, torch.float32), _t(u, torch.float32), want_probs=True)
    p, probs, tok, tprob = x.cpu().numpy(), probs.cpu().numpy(), tok.cpu().numpy(), tprob.cpu().numpy()
    for r, k in enumerate(ks):
        kth = np.sort(p[r])[::-1][k - 1]
        assert np.array_equal(probs[r] > 0, p[r] >= kth), f"k={k}: kept set is not {{p >= k-th largest p}}"
        if 39 <= k <= 42:
            assert set(np.flatnonzero(probs[r] > 0)) == set(above) | set(ties), f"k={k}: the tie group must be kept whole"
        assert probs[r][tok[r]] > 0 and tprob[r] == probs[r][tok[r]]
    assert tok[0] == above[-1]                               # k = 1: the maximum


@pytest.mark.parametrize("V", [1000, 32000])
def test_top_k_without_limit(V):
    """top_k <= 0, == V and > V all mean no limit: bit-identical to top_k = 0, with every token kept."""
    rng = np.random.default_rng(V + 1)
    lg = (rng.standard_normal(V) * 3).astype(F32)
    ks = [0, -1, -(2 ** 31), V, V + 1, 2 ** 31 - 1]
    n = len(ks)
    x = torch.from_numpy(lg).to(dev).expand(n, V).contiguous()
    tok, tprob, probs = ops.sample(x, _t(ks, torch.int32), _t([1.0] * n, torch.float32), _t([0.637] * n, torch.float32),
                                   want_probs=True)
    p, probs, tok, tprob = x.cpu().numpy(), probs.cpu().numpy(), tok.cpu().numpy(), tprob.cpu().numpy()
    assert np.array_equal(probs[0] > 0, p[0] > 0)
    for r in range(1, n):
        assert np.array_equal(probs[r], probs[0]) and tok[r] == tok[0] and tprob[r] == tprob[0], f"top_k={ks[r]}"


def _top_p_ok(p, kept, k, tp, V):
    """The kept set is {p >= thr} for a thr at or above the top-k threshold, and in float64 it is the smallest such set of
    largest p whose mass reaches tp of the top-k mass -- up to the rounding of the kernel's fp32 block sums (each adds
    ceil(V/1024) terms per thread, 5 shuffle levels and 32 warp partials, on both sides of the comparison)."""
    thr = p[kept].min()
    if not np.array_equal(kept, p >= thr):
        return "not a threshold set"
    srt = np.sort(p)[::-1]
    kth = srt[k - 1] if 0 < k < V else F32(0)
    if thr < kth:
        return f"threshold {thr} below the top-k threshold {kth}"
    p64 = p.astype(np.float64)
    need = float(F32(tp)) * p64[p >= kth].sum()
    delta = (-(-V // THREADS) + 40) * 2.0 ** -23
    if p64[p >= thr].sum() < need * (1 - delta):
        return f"kept mass {p64[p >= thr].sum()} short of {need}"
    if p64[p > thr].sum() >= need * (1 + delta):
        return f"not the smallest set: mass above the threshold {p64[p > thr].sum()} already reaches {need}"
    return None


@pytest.mark.parametrize("V", [1000, 32000, 152064])
def test_top_p_keeps_the_smallest_prefix_reaching_the_mass(V):
    rng = np.random.default_rng(V + 2)
    per = -(-V // THREADS)
    lg = rng.standard_normal(V).astype(F32)
    tops = _spread(V, 3, per, 10)
    lg[tops] = lg.max() + 2                                  # three exact maxima in different chunks
    rows = [(0, 0.1), (0, 0.5), (0, 0.9), (0, 0.99), (20, 0.95), (0, 1e-6), (7, 1e-6),
            (0, 0.0), (0, 5e-8), (0, -5e-8), (7, 0.0), (7, 5e-8), (0, 1.0), (7, 1.0)]
    n = len(rows)
    x = torch.from_numpy(lg).to(dev).expand(n, V).contiguous()
    tok, tprob, probs = ops.sample(x, _t([k for k, _ in rows], torch.int32), _t([tp for _, tp in rows], torch.float32),
                                   _t([0.637] * n, torch.float32), want_probs=True)
    p, probs, tok, tprob = x.cpu().numpy(), probs.cpu().numpy(), tok.cpu().numpy(), tprob.cpu().numpy()
    row = {r: i for i, r in enumerate(rows)}
    for i, (k, tp) in enumerate(rows):
        kept = probs[i] > 0
        assert kept[tok[i]] and tprob[i] == probs[i][tok[i]]
        if abs(F32(tp)) < 1e-7:                              # no top-p limit: the same bits as top_p = 1
            j = row[(k, 1.0)]
            assert np.array_equal(probs[i], probs[j]) and tok[i] == tok[j], f"top_k={k} top_p={tp}"
        elif tp == 1e-6:                                     # the maxima only
            assert set(np.flatnonzero(kept)) == set(tops), f"top_k={k} top_p=1e-6"
        elif tp < 1:
            err = _top_p_ok(p[i], kept, k, tp, V)
            assert err is None, f"top_k={k} top_p={tp}: {err}"


@pytest.mark.parametrize("V", [1000, 1025, 128256])
def test_top_k_1_takes_the_lowest_index_among_maxima(V):
    rng = np.random.default_rng(V + 3)
    per = -(-V // THREADS)
    lg = rng.standard_normal(V).astype(F32)
    tops = _spread(V, 3, per, 1)
    lg[tops] = 9.0
    u = np.array([0, 0.3, 0.999, BELOW_ONE], F32)
    n = len(u)
    x = torch.from_numpy(lg).to(dev).expand(n, V).contiguous()
    tok, tprob, probs = ops.sample(x, _t([1] * n, torch.int32), _t([1.0, 0.5, 1.0, 0.2], torch.float32), _t(u, torch.float32),
                                   want_probs=True)
    probs, tok, tprob = probs.cpu().numpy(), tok.cpu().numpy(), tprob.cpu().numpy()
    assert (tok == tops.min()).all(), (tok, tops)
    for r in range(n):
        assert set(np.flatnonzero(probs[r] > 0)) == set(tops) and tprob[r] == probs[r][tok[r]]


def test_masked_logits_are_never_drawn():
    V = 32000
    per = -(-V // THREADS)
    rng = np.random.default_rng(11)
    lg = (rng.standard_normal(V) * 3).astype(F32)
    lg[rng.random(V) < 0.7] = -np.inf
    lg[100 * per:300 * per] = -np.inf                        # whole masked chunks in the middle and at the end
    lg[900 * per:] = -np.inf
    masked = np.isneginf(lg)
    _, _, p, probs = _sample_copies(lg, np.zeros(1, F32), 0, 1.0)
    assert (p[masked] == 0).all() and (probs[masked] == 0).all()
    u, _ = Draw(p, probs > 0).probes()
    u = np.concatenate([u, rng.random(256).astype(F32)])
    tok, tprob, _, _ = _sample_copies(lg, u, 0, 1.0)
    assert not masked[tok].any()
    _check_draws(u, tok, tprob, p, probs, "masked row")
    # one finite logit: that token, with probability 1, whatever the uniform and filters
    one = np.full(V, -np.inf, F32)
    one[12345] = -3.0
    n = 4
    x = torch.from_numpy(one).to(dev).expand(n, V).contiguous()
    tok, tprob, probs = ops.sample(x, _t([0, 5, 1, 0], torch.int32), _t([1.0, 0.5, 1.0, 0.9], torch.float32),
                                   _t([0, 0.5, 0.9, BELOW_ONE], torch.float32), want_probs=True)
    assert (tok.cpu().numpy() == 12345).all() and (tprob.cpu().numpy() == 1.0).all()
    assert probs.cpu().numpy()[:, 12345].tolist() == [1.0] * n


@pytest.mark.parametrize("V", [1000, 32000])
def test_penalties_at_their_edges(V):
    rng = np.random.default_rng(V + 4)
    S = 300
    B = 6
    lg = (rng.standard_normal((B, V)) * 3).astype(F32)
    hist = rng.integers(0, V, (B, S)).astype(np.int32)
    hist[0, ::3] = -1                                        # ids outside [0, V) are ignored
    hist[0, 1::7] = V
    hist[0, 2::11] = 2 ** 31 - 1
    hl = np.array([S, 0, S, S, S, S], np.int32)              # hist_len 0, and hist_len equal to the stride
    hist[3] = 17                                             # one token 300 times, with a positive logit ...
    hist[5] = 23                                             # ... and with a negative one
    lg[3, 17], lg[5, 23] = 2.5, -1.5
    kw = dict(temperature=np.array([0.7, 1.0, 1.3, 1.0, 0.5, 2.0], F32), history=hist, hist_len=hl,
              repetition=np.array([1.3, 1.5, 1.2, 1.3, 1.4, 1.1], F32), presence=np.array([0.2, 0.5, 0, 0.4, 0.3, 0.1], F32),
              frequency=np.array([0.1, 0.2, 0.05, 0.01, 0.2, 0.02], F32),
              process=np.array([1, 1, 1, 1, 0, 1], np.uint8))          # row 4: do_sample false, nothing applied
    top_k, top_p, u = np.zeros(B, np.int32), np.ones(B, F32), rng.random(B).astype(F32)
    ws = torch.zeros(B, V, dtype=torch.int32, device=dev)

    def run():
        x = torch.from_numpy(lg).to(dev)
        tok, tprob, probs = ops.sample(x, _t(top_k, torch.int32), _t(top_p, torch.float32), _t(u, torch.float32),
                                       temperature=_t(kw["temperature"], torch.float32), history=_t(hist, torch.int32),
                                       hist_len=_t(hl, torch.int32), repetition=_t(kw["repetition"], torch.float32),
                                       presence=_t(kw["presence"], torch.float32), frequency=_t(kw["frequency"], torch.float32),
                                       process=_t(kw["process"], torch.uint8), count_ws=ws, want_probs=True)
        torch.cuda.synchronize()
        assert int(ws.abs().sum()) == 0, "count workspace not left clean"
        return x.cpu().numpy(), probs.cpu().numpy(), tok.cpu().numpy(), tprob.cpu().numpy()

    soft, probs, tok, tprob = run()
    _, _, esoft, eprobs = orc.sample(lg, top_k, top_p, u, **kw)
    np.testing.assert_allclose(soft, esoft, rtol=2e-4, atol=1e-9)
    np.testing.assert_allclose(probs, eprobs, rtol=1e-3, atol=1e-7)
    # the second call reuses the workspace the first one cleaned: the same bits
    soft2, probs2, tok2, tprob2 = run()
    assert np.array_equal(soft, soft2) and np.array_equal(probs, probs2) and np.array_equal(tok, tok2)
    assert np.array_equal(tprob.view(np.uint32), tprob2.view(np.uint32))
    # row 4 (process 0) is the plain softmax, row 1 (hist_len 0) only sees its temperature
    for r in (1, 4):
        _, _, e, _ = orc.sample(lg[r:r + 1], top_k[:1], top_p[:1], u[:1], temperature=kw["temperature"][r:r + 1],
                                process=kw["process"][r:r + 1])
        np.testing.assert_allclose(soft[r], e[0], rtol=2e-4, atol=1e-9)


def _batch_inputs(B, V, seed):
    rng = np.random.default_rng(seed)
    S = 64
    return dict(
        lg=(rng.standard_normal((B, V)) * 3).astype(F32),
        top_k=rng.choice([0, 1, 5, 50, 1000], B).astype(np.int32),
        top_p=rng.choice([1.0, 0.95, 0.7, 0.3, 0.0], B).astype(F32),
        u=rng.random(B).astype(F32),
        temperature=(rng.random(B) + 0.3).astype(F32),
        history=rng.integers(-2, V + 2, (B, S)).astype(np.int32),
        hist_len=rng.integers(0, S + 1, B).astype(np.int32),
        repetition=rng.choice([1.0, 1.2], B).astype(F32),
        presence=rng.choice([0.0, 0.3], B).astype(F32),
        frequency=rng.choice([0.0, 0.1], B).astype(F32),
        process=(rng.random(B) < 0.9).astype(np.uint8))


def _run_batch(d, rows=slice(None)):
    x = torch.from_numpy(np.ascontiguousarray(d["lg"][rows])).to(dev)
    ws = torch.zeros_like(x, dtype=torch.int32)
    dt = dict(top_k=torch.int32, history=torch.int32, hist_len=torch.int32, process=torch.uint8)
    a = {k: _t(np.ascontiguousarray(v[rows]), dt.get(k, torch.float32)) for k, v in d.items() if k != "lg"}
    tok, tprob, probs = ops.sample(x, a.pop("top_k"), a.pop("top_p"), a.pop("u"), count_ws=ws, want_probs=True, **a)
    return x, probs, tok, tprob


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)


def test_rows_are_independent_and_the_op_deterministic():
    B, V = 1024, 32000
    d = _batch_inputs(B, V, 5)
    full = _run_batch(d)
    again = _run_batch(d)
    torch.cuda.synchronize()
    for a, b in zip(full, again):
        assert _same_bits(a, b), "the same call gave different bits"
    alone = [_run_batch(d, slice(r, r + 1)) for r in range(B)]
    torch.cuda.synchronize()
    for i, name in enumerate(("probabilities", "probs_out", "token", "token_prob")):
        one = torch.cat([a[i] for a in alone])
        diff = [r for r in range(B) if not _same_bits(one[r], full[i][r])]
        assert not diff, f"{name} of rows {diff[:8]} differ when the row runs alone"


def test_sample_after_an_lm_head_gemm_under_pdl_in_a_graph():
    """fp16 lm_head GEMM -> fp32 cast -> sample, with PDL on and captured in a CUDA graph: the tokens, their probabilities
    and the probabilities left in the logits are those of the same chain run eagerly without PDL."""
    B, K, V = 32, 4096, 128256
    gen = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(B, K, generator=gen, device=dev).half()
    w = ops.pack_f16((torch.randn(K, V, generator=gen, device=dev) * 0.05).half())
    ws = ops.gemm_workspace(B, [(K, V)], dev)
    y = torch.empty(B, V, dtype=torch.float16, device=dev)
    logits = torch.empty(B, V, dtype=torch.float32, device=dev)
    rng = np.random.default_rng(7)
    top_k = _t(rng.choice([0, 1, 40, 1000], B), torch.int32)
    top_p = _t(rng.choice([1.0, 0.9, 0.5], B), torch.float32)
    u = _t(rng.random(B), torch.float32)
    temp = _t(rng.random(B) + 0.5, torch.float32)

    def chain(pdl):
        ops.wo_gemm(x, w, ws, out=y, pdl=pdl)
        logits.copy_(y)
        return ops.sample(logits, top_k, top_p, u, temperature=temp)

    tok, tprob, _ = chain(False)
    torch.cuda.synchronize()
    ref = (tok.clone(), tprob.clone(), logits.clone())
    try:
        ops.set_pdl(True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain(True)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gtok, gtprob, _ = chain(True)
        y.fill_(float("nan"))
        logits.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)
    assert torch.equal(gtok, ref[0]), "tokens differ under PDL"
    assert _same_bits(gtprob, ref[1]) and _same_bits(logits, ref[2])
