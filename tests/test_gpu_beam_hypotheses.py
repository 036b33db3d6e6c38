"""GPU tests (H100) of the finished-hypothesis set of beam search: b200_beam_hypotheses_update / _finalize against the float64
reference (tests/beam_hyps_oracle.py) over seeded candidate streams, their bits under CUDA-graph replay with PDL, and
DecodeStep's beam mode with an eos_id: the set after every step, beam_results, a re-score of every returned path through
plain steps, early stopping, and the step without an eos_id."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep  # noqa: E402
from tests.beam_hyps_oracle import FALSE, NEVER, TRUE, Hyps, check_finalize, check_state, hyp_score, parse_state  # noqa: E402

DEV = torch.device("cuda")
EOS = 7
ALPHAS = [0.0, 1.0, 2.0, -1.0, 0.5]


def _gen_paths(hist, hl, gen_start=1):
    """Each row's generated tokens: history[row][gen_start : hist_len] (hist_len clamped to the stride)."""
    return [hist[r, gen_start:min(int(hl[r]), hist.shape[1])].tolist() for r in range(hist.shape[0])]


def _rows(rng, R, stride):
    """Token histories [R, stride] and lengths, some without a generated token and some past the stride (clamped)."""
    return rng.integers(0, 1000, (R, stride)).astype(np.int32), rng.integers(0, stride + 4, R).astype(np.int32)


def _stream(B, W, steps, stride, seed):
    """Seeded update inputs: ranked candidate scores on a coarse grid (exact ties), some -inf, EOS at 40 % of the ranks."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        K = 2 * W
        grid = -rng.integers(1, 16, (B, K)).astype(np.float32) / 4
        grid[rng.random((B, K)) < 0.08] = -np.inf
        hist, hl = _rows(rng, B * W, stride)
        out.append(dict(cand_token=np.where(rng.random((B, K)) < 0.4, EOS, rng.integers(0, 40, (B, K))).astype(np.int32),
                        cand_parent=rng.integers(0, W, (B, K)).astype(np.int32),
                        cand_score=-np.sort(-grid, axis=1), history=hist, hist_len=hl))
    return out


def _to_dev(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in d.items()}


@pytest.mark.parametrize("W", [1, 4, 16, 32])
def test_update_and_finalize_vs_reference(W):
    B, stride, max_len = 128 // W, 24, 16                   # paths of up to 24 tokens: some are cut to max_len
    steps = 64 if W <= 4 else 24
    stream = _stream(B, W, steps, stride, seed=W)
    dev = [_to_dev(s) for s in stream]
    alphas = [ALPHAS[b % len(ALPHAS)] for b in range(B)]
    modes = [(FALSE, NEVER, TRUE)[b % 3] for b in range(B)]
    lp = torch.tensor(alphas, dtype=torch.float32, device=DEV)
    es = torch.tensor(modes, dtype=torch.int32, device=DEV)
    state = ops.beam_hypotheses_state(B, W, max_len, DEV)
    done = torch.zeros(B, dtype=torch.int32, device=DEV)
    ref = [Hyps(W, max_len) for _ in range(B)]
    rng = np.random.default_rng(100 + W)
    live_cum = -rng.integers(1, 48, (B, W)).astype(np.float32) / 4
    live_cum[rng.random((B, W)) < 0.1] = -np.inf
    live_hist, live_hl = _rows(rng, B * W, stride)
    live = _to_dev(dict(cum=live_cum, history=live_hist, hist_len=live_hl))
    live_paths = _gen_paths(live_hist, live_hl)
    ties = exact = 0
    for t, (s, d) in enumerate(zip(stream, dev)):
        ops.beam_hypotheses_update(d, d["history"], d["hist_len"], EOS, lp, es, state, done, max_len, gen_start=1)
        paths = _gen_paths(s["history"], s["hist_len"])
        for b, h in enumerate(ref):
            if not h.done and len(h.slots) == W:                # candidates at exactly the worst score (must not enter)
                ties += sum(1 for r in range(W) if s["cand_token"][b, r] == EOS and np.isfinite(s["cand_score"][b, r]) and
                            hyp_score(s["cand_score"][b, r], len(paths[b * W + s["cand_parent"][b, r]]) + 1, alphas[b]) == h.worst())
            h.update(s["cand_token"][b], s["cand_parent"][b], s["cand_score"][b], paths[b * W:(b + 1) * W], EOS, alphas[b], modes[b])
        got, dn = parse_state(state.cpu().numpy(), B, W, max_len), done.cpu().numpy()
        for b in range(B):
            exact += check_state(got[b], ref[b], dn[b], alphas[b], f"W{W} step {t} request {b}")
        if t in (steps // 2, steps - 1):
            before = state.clone()
            for n in range(1, W + 1):
                out = ops.beam_hypotheses_finalize(state, done, live["cum"], live["history"], live["hist_len"], n, max_len, lp,
                                                   gen_start=1)
                o = {k: v.cpu().numpy() for k, v in out.items()}
                for b in range(B):
                    e = ref[b].finalize(n, live_cum[b], live_paths[b * W:(b + 1) * W], alphas[b])
                    check_finalize({k: v[b] for k, v in o.items()}, e, f"W{W} step {t} n {n} request {b}")
            assert torch.equal(state, before), "finalize modified the state"
    assert exact >= 0.9 * steps * B, (exact, steps * B)
    assert ties > 0 or W == 1, "no candidate tied the worst score"     # at W 1 a full set is nearly always done
    assert any(h.next_order > W for h in ref), "no hypothesis was replaced"
    assert int(done.sum()) > 0, "no request was done"

    # the same stream under a CUDA graph with PDL: the same state bytes and outputs, bit for bit
    eager = [state.clone(), done.clone()] + list(ops.beam_hypotheses_finalize(state, done, live["cum"], live["history"],
                                                                              live["hist_len"], W, max_len, lp, gen_start=1).values())
    st2, dn2 = torch.empty_like(state), torch.empty_like(done)
    out2 = ops.beam_hypotheses_finalize(state, done, live["cum"], live["history"], live["hist_len"], W, max_len, lp, gen_start=1)

    def run():
        st2.zero_()
        dn2.zero_()
        for d in dev:
            ops.beam_hypotheses_update(d, d["history"], d["hist_len"], EOS, lp, es, st2, dn2, max_len, gen_start=1)
        ops.beam_hypotheses_finalize(st2, dn2, live["cum"], live["history"], live["hist_len"], W, max_len, lp, gen_start=1, out=out2)
    ops.set_pdl(True)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            run()
        for _ in range(2):
            for v in list(out2.values()) + [st2, dn2]:
                v.fill_(-7)
            graph.replay()
            torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(eager, [st2, dn2] + list(out2.values()))), "graph replay with PDL differs"
    finally:
        ops.set_pdl(False)


# ---------------------------------------------------------------------------------------------------- decode step
W, CTX, STEPS = 4, 64, 30          # tokens_per_block 16: every row crosses a page boundary within the 30 steps


def _pick_eos(cfg, seed, fill):
    """An EOS from a first run of the same seeded step without EOS: the token most often ranked below W. With fill, the first
    of the 32 most frequent ones with which some request's set fills within the steps (early stopping True sets done)."""
    model = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=seed, beam_width=W, max_new_tokens=STEPS)
    counts = {}
    for _ in range(STEPS):
        model.run()
        torch.cuda.synchronize()
        for tok in model.beam_out["cand_token"][:, :W].cpu().view(-1).tolist():
            counts[tok] = counts.get(tok, 0) + 1
    del model
    ranked = sorted(counts, key=lambda k: (-counts[k], k))
    if not fill:
        return ranked[0]
    for e in ranked[:32]:
        trial = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=seed, beam_width=W, max_new_tokens=STEPS, eos_id=e,
                           early_stopping=True)
        for _ in range(STEPS):
            trial.run()
        if int(trial.done.sum()) > 0:
            return e
    pytest.fail(f"none of the tokens {ranked[:32]} fills a hypothesis set in {STEPS} steps")


def _rescore(cfg, seed, beam, kv0, res, ids0):
    """Every returned hypothesis fed through plain (greedy) steps as forced inputs, on a cache that starts as a copy of the
    beam step's prompt: the float64 log-softmax of each of its tokens, summed, must match its cum within 1e-2 per token."""
    B = beam.requests
    plain = DecodeStep(cfg, B * W, CTX, DEV, ragged=True, seed=seed)
    plain.block_ids_h.copy_(beam.block_ids_h)
    plain.seq_lens_h.copy_(beam.seq_lens_h)
    for Lp, kv in zip(plain.layers, kv0):
        Lp["kv"].copy_(kv)
    n = res["len"].shape[1]
    full = [[int(ids0[b * W])] + res["tokens"][b, k, :max(int(res["len"][b, k]), 0)].tolist() for b in range(B) for k in range(n)]
    score = np.zeros(len(full))
    for t in range(max(len(p) for p in full) - 1):
        plain.ids_h.copy_(torch.tensor([p[min(t, len(p) - 1)] for p in full], dtype=torch.int32))
        plain.seq_lens_h.copy_(beam.seq_lens_h + t)
        plain.upload_inputs()
        plain.run()
        torch.cuda.synchronize()
        x = plain.logits.double().cpu().numpy()
        m = x.max(1, keepdims=True)
        ls = x - m - np.log(np.exp(x - m).sum(1, keepdims=True))
        for j, p in enumerate(full):
            if t + 1 < len(p):
                score[j] += ls[j, p[t + 1]]
    cum = res["cum"].numpy().reshape(-1).astype(np.float64)
    lens = res["len"].numpy().reshape(-1)
    have = lens > 0
    assert (np.abs(score - cum)[have] <= 1e-2 * lens[have]).all(), (score, cum, lens)


STEP = [("int4", "eager", (1.0, 0.0), (False, "never")), ("f16", "eager", (2.0, -1.0), ("never", False)),
        ("int4", "graph pdl", (1.0, 2.0), (True, True)), ("f16", "graph pdl", (0.5, 1.0), (False, True))]


@pytest.mark.parametrize("case", STEP, ids=[f"{q} {m} alpha {a} early {e}" for q, m, a, e in STEP])
def test_step_hypotheses_vs_reference(case):
    quant, mode, alphas, early = case
    cfg, seed = dataclasses.replace(TINY, quant=quant), 4
    e = _pick_eos(cfg, seed, fill=True in early)
    model = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=seed, pdl="pdl" in mode, beam_width=W, max_new_tokens=STEPS, eos_id=e,
                       length_penalty=list(alphas), early_stopping=list(early))
    B, R = model.requests, model.B
    modes = [NEVER if m == "never" else int(m) for m in early]
    kv0 = [L["kv"].clone() for L in model.layers]
    ids0 = model.ids_h.clone()
    seq0 = model.seq_lens_h.clone().long()
    assert ((seq0 + STEPS) // cfg.tokens_per_block > seq0 // cfg.tokens_per_block).all(), "no page crossing"
    stride = 16 + 16 * W + 4 * W * STEPS
    try:
        if "graph" in mode:
            model.capture()
        model.upload_inputs()
        ref = [Hyps(W, STEPS) for _ in range(B)]
        paths = [[] for _ in range(R)]                        # each row's generated tokens, by its next_parent ancestry
        frozen = [None] * B
        for t in range(STEPS):
            torch.cuda.synchronize()
            hist, hl = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
            assert _gen_paths(hist, hl) == paths, f"step {t}: history is not the ancestry"
            model.replay() if "graph" in mode else model.run()
            torch.cuda.synchronize()
            o = {k: v.cpu().numpy() for k, v in model.beam_out.items()}
            for b, h in enumerate(ref):
                h.update(o["cand_token"][b], o["cand_parent"][b], o["cand_score"][b], paths[b * W:(b + 1) * W], e, alphas[b], modes[b])
            raw = model.hyp_state.cpu()
            got, dn = parse_state(raw.numpy(), B, W, STEPS), model.done.cpu().numpy()
            for b in range(B):
                check_state(got[b], ref[b], dn[b], alphas[b], f"{case} step {t} request {b}")
                if modes[b] == TRUE:
                    assert bool(dn[b]) == (got[b]["count"] == W), f"step {t} request {b}: done is not 'the set is full'"
                if frozen[b] is not None:
                    assert torch.equal(raw[b * stride:(b + 1) * stride], frozen[b]), f"step {t} request {b}: changed after done"
                elif dn[b]:
                    frozen[b] = raw[b * stride:(b + 1) * stride].clone()
            par = (np.arange(R) // W * W + o["next_parent"].reshape(-1)).tolist()
            paths = [paths[par[j]] + [int(o["next_token"].reshape(-1)[j])] for j in range(R)]
        assert sum(h.next_order for h in ref) > 0, f"EOS {e}: no hypothesis was inserted"
        if TRUE in modes:
            assert any(frozen[b] is not None for b in range(B) if modes[b] == TRUE), "no request stopped early"
        cum = model.beam_cum.cpu().numpy()
        hist, hl = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
        assert _gen_paths(hist, hl) == paths
        for n in range(1, W + 1):
            res = model.beam_results(n)
            for b in range(B):
                check_finalize({k: v[b].numpy() for k, v in res.items()}, ref[b].finalize(n, cum[b], paths[b * W:(b + 1) * W],
                                                                                         alphas[b]), f"{case} n {n} request {b}")
        # the reference was fed each row's next_parent ancestry, not the device history: equal paths are the beams' ancestry
        _rescore(cfg, seed, model, kv0, model.beam_results(W), ids0)
    finally:
        ops.set_pdl(False)


def test_without_eos_the_step_is_unchanged():
    cfg = dataclasses.replace(TINY, quant="int4")
    a = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=5, beam_width=W, max_new_tokens=8)
    b = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=5, beam_width=W, max_new_tokens=8, eos_id=None, length_penalty=2.0,
                   early_stopping=True)
    c = DecodeStep(cfg, 2, CTX, DEV, ragged=True, seed=5, beam_width=W, max_new_tokens=8, eos_id=3)
    la, lb, lc = a.launches_per_step(), b.launches_per_step(), c.launches_per_step()
    assert la == lb and lc == la + 1, (la, lb, lc)
    assert not hasattr(b, "hyp_state")
    for _ in range(6):
        torch.cuda.synchronize()
        assert torch.equal(a.logits, b.logits)
        assert all(torch.equal(a.beam_out[k], b.beam_out[k]) for k in a.beam_out)
        n = int(a.hist_len.max())
        assert torch.equal(a.beam_cum, b.beam_cum) and torch.equal(a.hist_len, b.hist_len)
        assert torch.equal(a.hist[:, :n], b.hist[:, :n])
        a.run()
        b.run()
