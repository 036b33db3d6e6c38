"""GPU tests (H100) of sampled decoding: b200_token_logprobs against the float64 reference (tests/logprob_oracle.py) and its
bits under CUDA-graph replay with PDL; DecodeStep's sampling mode step by step against oracle_step and the sampler oracle
(pinned to the reference's CudaSamplerTest vectors) on the step's own logits, params, history and uniforms; and sampled
verification of speculative tokens against spec_verify_np on the step's own probabilities and uniforms."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams, sampling_uniforms  # noqa: E402
from tests.beam_oracle import banned_np  # noqa: E402
from tests.logprob_oracle import log_softmax_np, token_logprobs_np  # noqa: E402
from tests.spec_oracle import spec_verify_np  # noqa: E402
from tests.step_oracle import bits, check_logits, device_state, oracle_step  # noqa: E402

DEV = torch.device("cuda")
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}


def _tol(lp):
    return 1e-5 * (1.0 + np.abs(lp))


def check_logprobs(got, exp, top_n):
    """token_logprob and every top_logprobs rank within 1e-5 * (1 + |lp|) of the float64 reference; top ids equal at every rank
    whose reference value is clear of its neighbours by that bound, and at exact ties (both take the lower id first)."""
    if "token_logprob" in exp:
        e, g = exp["token_logprob"], got["token_logprob"].astype(np.float64)
        fin = np.isfinite(e)
        assert (np.isneginf(g) == np.isneginf(e)).all() and (np.isnan(g) == np.isnan(e)).all()
        assert (np.abs(g[fin] - e[fin]) <= _tol(e[fin])).all(), np.abs(g - e)[fin].max()
    if top_n == 0:
        return
    e, g, rs = exp["top_logprobs"], got["top_logprobs"].astype(np.float64), exp["ranked"]
    fin = np.isfinite(e)
    assert (np.isneginf(g) == np.isneginf(e)).all()
    assert (np.abs(g[fin] - e[fin]) <= _tol(e[fin])).all(), np.abs(g - e)[fin].max()

    def clear(a, c):
        return (np.isneginf(a) and np.isneginf(c)) or a == c or abs(a - c) > _tol(a)
    for r in range(e.shape[0]):
        for k in range(top_n):
            if clear(rs[r, k], rs[r, k + 1]) and (k == 0 or clear(rs[r, k - 1], rs[r, k])):
                assert got["top_ids"][r, k] == exp["top_ids"][r, k], (r, k, got["top_ids"][r], exp["top_ids"][r])


ROWS = {64: 128, 1000: 1, 32000: 37, 128256: 9, 152064: 3}


def _rows_case(rows, V, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, V, generator=g) * 3.0
    x[0, ::7] = -float("inf")                                        # masked logits
    if rows > 1:
        x[1] = 0.25                                                  # all equal
    if rows > 2:
        x[2, V // 2:] = x[2, : V - V // 2]                          # exact duplicates: every value twice
    return x.to(dtype)


@pytest.mark.parametrize("top_n", [0, 1, 5, 20])
@pytest.mark.parametrize("V", list(ROWS))
@pytest.mark.parametrize("dt", list(DTYPES))
def test_logprobs_vs_float64_reference(dt, V, top_n):
    rows = ROWS[V]
    x = _rows_case(rows, V, DTYPES[dt], seed=V + top_n)
    tok = torch.randint(0, V, (rows,), generator=torch.Generator().manual_seed(V), dtype=torch.int32)
    tok[0] = 0                                                       # a masked logit: -inf
    out = ops.token_logprobs(x.to(DEV), top_n, tokens=tok.to(DEV))
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    exp = token_logprobs_np(x.double().numpy(), top_n, tokens=tok.numpy())
    assert np.isneginf(got["token_logprob"][0])
    check_logprobs(got, exp, top_n)
    if top_n and rows > 1:                                           # the all-equal row: ids 0.. in order, all -log V
        np.testing.assert_array_equal(got["top_ids"][1], np.arange(top_n))
    if top_n and rows > 2:                                           # duplicates: each value's lower id first
        ids = got["top_ids"][2]
        assert all(ids[k] < ids[k + 1] for k in range(0, top_n - 1, 2) if got["top_logprobs"][2, k] == got["top_logprobs"][2, k + 1])


def test_logprobs_give_the_same_bits_under_graph_replay_with_pdl():
    rows, V, n = 32, 128256, 20
    src = _rows_case(rows, V, torch.float16, seed=5).to(DEV)
    tok = torch.randint(0, V, (rows,), generator=torch.Generator().manual_seed(1), dtype=torch.int32).to(DEV)
    x = torch.empty_like(src)
    ws = ops.token_logprobs_workspace(rows, V, n, DEV)
    out = dict(token_logprob=torch.empty(rows, device=DEV), top_ids=torch.empty(rows, n, dtype=torch.int32, device=DEV),
               top_logprobs=torch.empty(rows, n, device=DEV))

    def run():
        x.copy_(src)
        ops.token_logprobs(x, n, tokens=tok, workspace=ws, out=out)

    def snap():
        torch.cuda.synchronize()
        return [v.clone() for v in out.values()]
    run()
    ref = snap()
    run()
    assert all(torch.equal(a, b) for a, b in zip(ref, snap())), "repeated eager calls differ"
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
        for _ in range(3):
            for v in out.values():
                v.fill_(-7)
            graph.replay()
            assert all(torch.equal(a, b) for a, b in zip(ref, snap())), "graph replay with PDL differs"
    finally:
        ops.set_pdl(False)
    assert int(ws[:4 * rows].view(torch.int32).abs().sum()) == 0, "arrival counters not reset"
    check_logprobs({k: v.cpu().numpy() for k, v in out.items()},
                   token_logprobs_np(src.double().cpu().numpy(), n, tokens=tok.cpu().numpy()), n)


# ---------------------------------------------------------------------------------------------------- decode step
# request 0: top_k 1 (greedy); 1: repetition 2 + presence 1, certain to move every history logit; 2: frequency; 3: top-k + top-p
PARAMS = SamplingParams(temperature=[0.7, 1.0, 1.3, 0.9], top_k=[1, 50, 0, 20], top_p=[1.0, 0.9, 0.8, 0.95],
                        repetition=[1.0, 2.0, 1.0, 1.3], presence=[0.0, 1.0, 0.0, 0.0], frequency=[0.0, 0.0, 0.5, 0.0], seed=11)
STEP = [("int4", "eager", 0), ("f16", "eager", 2), ("int4", "graph pdl", 2), ("f16", "graph pdl", 0)]


def _draw_ok(tok, etok, probs, u):
    """Equal tokens, or a draw within 1e-6 * total of a CDF boundary of the oracle's kept distribution."""
    if tok == etok:
        return True
    cdf = np.cumsum(probs.astype(np.float64))
    return float(np.min(np.abs(cdf - u * cdf[-1]))) < 1e-6 * cdf[-1]


@pytest.mark.parametrize("case", STEP, ids=[f"{q} {m} ngram {n}" for q, m, n in STEP])
def test_sampling_step_vs_oracles(case):
    quant, mode, ngram = case
    cfg = dataclasses.replace(TINY, quant=quant)
    steps, n_lp = 6, 5
    model = DecodeStep(cfg, 4, 40, DEV, keep_reference=True, ragged=True, seed=3, pdl="pdl" in mode, sampling=PARAMS,
                       logprobs=n_lp, max_new_tokens=8, no_repeat_ngram=ngram)
    R, V, T = model.B, model.vocab, cfg.tokens_per_block
    p = {k: np.asarray(getattr(PARAMS, k), np.float32) for k in ("temperature", "top_p", "repetition", "presence", "frequency")}
    p["top_k"] = np.asarray(PARAMS.top_k, np.int32)
    seq0 = model.seq_lens_h.clone().long()
    assert ((seq0 + steps) // T > seq0 // T).any(), "no page crossing in this run"
    try:
        if "graph" in mode:
            model.capture()
        model.upload_inputs()
        torch.cuda.synchronize()
        paths = [[int(t)] for t in model.ids.cpu().tolist()]
        cum = np.zeros(R, np.float64)
        moved = 0
        for t in range(steps):
            torch.cuda.synchronize()
            state, kv_before = device_state(model), [bits(L["kv"]) for L in model.layers]
            hist, hist_len = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
            model.replay() if "graph" in mode else model.run()
            torch.cuda.synchronize()
            raw = model.logits.float().cpu().numpy()
            check_logits(raw, oracle_step(state, kv_before))
            u = model.uniform.cpu()
            assert torch.equal(u, sampling_uniforms(PARAMS.seed, t, R)), f"step {t}: uniforms"
            lg = raw.copy()
            if ngram:
                for r, b in enumerate(banned_np(hist, hist_len, [ngram] * R, V)):
                    lg[r, b] = -np.inf
            etok, _, esoft, eprobs = orc.sample(lg, p["top_k"], p["top_p"], u.numpy(), temperature=p["temperature"], history=hist,
                                                hist_len=hist_len, repetition=p["repetition"], presence=p["presence"],
                                                frequency=p["frequency"])
            tok, tprob = model.next_ids.cpu().numpy(), model.token_prob.cpu().numpy()
            soft = model.samp_logits.cpu().numpy()
            np.testing.assert_allclose(soft, esoft, rtol=2e-4, atol=1e-9)
            for r in range(R):
                assert _draw_ok(tok[r], etok[r], eprobs[r], float(u[r])), f"step {t} row {r}: {tok[r]} vs oracle {etok[r]}"
            # penalties certain to fire (request 1: repetition 2, presence 1) move exactly the history tokens' logits
            h1 = np.unique(hist[1, :hist_len[1]])
            d = np.log(np.maximum(soft[1].astype(np.float64), 1e-300)) - raw[1].astype(np.float64)   # temperature 1: not applied
            other = np.ones(V, bool)
            other[h1] = False
            c = np.median(d[other])
            assert np.abs(d[other] - c).max() < 1e-3 and (np.abs(d[h1] - c) > 0.5).all(), f"step {t}: penalised set"
            # cum_log_probs is the running sum of log token_prob; the history rows are the emitted tokens
            cum += np.log(tprob.astype(np.float64))
            np.testing.assert_allclose(model.cum_log_probs.cpu().numpy(), cum, rtol=1e-5)
            moved += int((tok != np.array([q[-1] for q in paths])).sum())
            paths = [paths[r] + [int(tok[r])] for r in range(R)]
            h, hl = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
            for r in range(R):
                assert hl[r] == len(paths[r]) and h[r, :hl[r]].tolist() == paths[r], f"step {t} row {r}: history"
            assert model.ids.cpu().tolist() == tok.tolist()
            assert (model.seq_lens.cpu().long() == seq0 + t + 1).all()
            # log-probs of the raw lm_head output
            exp = token_logprobs_np(raw, n_lp, tokens=tok)
            check_logprobs({k: v.cpu().numpy() for k, v in model.lp_out.items()}, exp, n_lp)
        assert moved > 0
        with pytest.raises(ValueError, match="max_new_tokens"):
            for _ in range(3):
                model.replay() if "graph" in mode else model.run()
    finally:
        ops.set_pdl(False)


def test_top_k_one_rows_are_the_greedy_steps_tokens():
    cfg = dataclasses.replace(TINY, quant="int4")
    samp = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=8, sampling=PARAMS, max_new_tokens=8)
    greedy = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=8)
    greedy.seq_lens_h.copy_(samp.seq_lens_h)
    greedy.upload_inputs()
    for m in (samp, greedy):
        m.run()
    torch.cuda.synchronize()
    assert torch.equal(samp.logits, greedy.logits)
    assert int(samp.next_ids[0]) == int(greedy.next_ids[0])


@pytest.mark.parametrize("q_len", [2, 4])
@pytest.mark.parametrize("mode", ["eager", "graph pdl"])
def test_sampled_verification_vs_reference(q_len, mode):
    cfg = dataclasses.replace(TINY, quant="int4")
    sp = SamplingParams(temperature=[0.5, 1.0, 1.0, 2.0], top_k=[0, 50, 5, 0], top_p=[1.0, 0.9, 1.0, 0.7], seed=5)
    model = DecodeStep(cfg, 4, 40, DEV, keep_reference=True, ragged=True, seed=4, pdl="pdl" in mode, sampling=sp, q_len=q_len,
                       logprobs=3)
    R = model.B * q_len
    g = torch.Generator().manual_seed(q_len)
    try:
        if "graph" in mode:
            model.capture()
        for t in range(3):
            model.ids_h[:, 1:] = torch.randint(0, cfg.vocab, (model.B, q_len - 1), generator=g, dtype=torch.int32)
            model.upload_inputs()
            torch.cuda.synchronize()
            kv_before = [bits(L["kv"]) for L in model.layers]
            state = device_state(model)
            model.replay() if "graph" in mode else model.run()
            torch.cuda.synchronize()
            raw = model.logits.float().cpu().numpy()
            check_logits(raw, oracle_step(state, kv_before))
            u = model.uniform.cpu()
            assert torch.equal(u, sampling_uniforms(sp.seed, 0, 2 * R)), "uniforms restart with upload_inputs()"
            rep = lambda v, dt: np.repeat(np.asarray(v, dt), q_len)  # noqa: E731
            _, _, _, eprobs = orc.sample(raw, rep(sp.top_k, np.int32), rep(sp.top_p, np.float32), u[:R].numpy(),
                                         temperature=rep(sp.temperature, np.float32))
            tp = model.target_probs.cpu().numpy()
            np.testing.assert_allclose(tp.reshape(R, -1), eprobs, rtol=1e-3, atol=1e-7)
            eo, ea = spec_verify_np(model.ids_h[:, 1:].numpy(), target_probs=tp, uniform=u[R:].numpy().reshape(model.B, q_len))
            np.testing.assert_array_equal(model.accepted.cpu().numpy(), ea)
            np.testing.assert_array_equal(model.out_tokens.cpu().numpy(), eo)
            check_logprobs({k: v.cpu().numpy() for k, v in model.lp_out.items()},
                           token_logprobs_np(raw, 3, tokens=model.next_ids.cpu().numpy()), 3)
    finally:
        ops.set_pdl(False)


def test_sampled_verification_accepts_near_greedy_drafts():
    """Drafts from a plain sampled run at near-zero temperature (one-hot kept sets): a verification step on an identical model
    accepts all of them wherever every plain step's top-2 margin is clear of the logit error."""
    cfg, k = dataclasses.replace(TINY, quant="int4"), 3
    cold = SamplingParams(temperature=1e-4, seed=2)
    plain = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2, sampling=cold, max_new_tokens=8)
    spec = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2, sampling=cold, q_len=k + 1)
    plain.seq_lens_h.copy_(spec.seq_lens_h)
    plain.ids_h.copy_(spec.ids_h[:, 0])
    plain.upload_inputs()
    toks, logits = [plain.ids_h.clone()], []
    for _ in range(k + 1):
        plain.run()
        torch.cuda.synchronize()
        logits.append(plain.logits.float().cpu().numpy())
        toks.append(plain.next_ids.cpu())
    spec.ids_h.copy_(torch.stack(toks[:k + 1], dim=1))
    spec.upload_inputs()
    spec.run()
    torch.cuda.synchronize()
    got = spec.logits.float().cpu().numpy().reshape(spec.B, k + 1, -1)
    exp = np.stack(logits, axis=1)
    err = check_logits(got, exp)
    srt = np.sort(exp, axis=-1)
    sure = ((srt[..., -1] - srt[..., -2]) > 2 * err + 1e-3).all(axis=1)
    assert sure.any(), "no sequence with a clear margin at every step"
    acc, out = spec.accepted.cpu().numpy(), spec.out_tokens.cpu().numpy()
    assert (acc[sure] == k).all(), acc
    np.testing.assert_array_equal(out[sure, :k], torch.stack(toks[1:k + 1], dim=1).numpy()[sure])
    np.testing.assert_array_equal(out[sure, k], toks[k + 1].numpy()[sure])


def test_log_softmax_reference_matches_torch():
    x = torch.randn(3, 1000, dtype=torch.float64)
    np.testing.assert_allclose(log_softmax_np(x.numpy()), torch.log_softmax(x, -1).numpy(), rtol=1e-12, atol=1e-12)
