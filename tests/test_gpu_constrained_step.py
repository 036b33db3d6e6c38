"""GPU tests (H100) of constrained decoding in the decode step: every ending (greedy, greedy verification, sampling with min-p,
sampled verification, beam) emits only tokens its row's mask allows, the logits it picks from are -inf where masked and
within the whole-step tolerance of tests/step_oracle.py elsewhere, a single allowed token or a +1e4 bias forces a token, a
host-side toy grammar drives graph replays without a violation, an all-ones mask changes no bit, and the constraints cost
one launch per step. TINY config, int4 and f16 weights, eager and graph + PDL, ragged lengths across page boundaries."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams  # noqa: E402
from tests.constrain_oracle import allowed  # noqa: E402
from tests.step_oracle import bits, check_logits, device_state, oracle_step  # noqa: E402

DEV = torch.device("cuda")
SP = SamplingParams(temperature=[0.8, 1.0, 1.2, 0.9], top_k=[0, 50, 0, 20], top_p=[1.0, 0.9, 0.95, 1.0],
                    min_p=[0.0, 0.05, 0.1, 0.0], seed=4)
# q_len 6: the verification steps' last tokens cross a page boundary (positions 31..36 of a 37-token sequence)
MODES = dict(greedy={}, verify=dict(q_len=6), sampling=dict(sampling=SP, max_new_tokens=8),
             sampled_verify=dict(sampling=SP, q_len=6), beam=dict(beam_width=4, max_new_tokens=8))


def pack(ok: np.ndarray) -> np.ndarray:
    """bool [rows, V] (V a multiple of 32) -> int32 [rows, V / 32] in xgrammar's layout (bit t & 31 of word t >> 5)."""
    return np.packbits(ok, axis=1, bitorder="little").view(np.int32)


def build(mode, quant="int4", run="eager", ctx=40, seed=5, **kw):
    cfg = dataclasses.replace(TINY, quant=quant)
    return DecodeStep(cfg, 4, ctx, DEV, ragged=True, seed=seed, pdl="pdl" in run, token_bitmask=True, logit_bias_capacity=64,
                      **MODES[mode], **kw)


def go(model, run):
    model.replay() if "graph" in run else model.run()
    torch.cuda.synchronize()


def emitted(model, mode):
    """(logits row, token) of every token the step emitted."""
    if mode in ("verify", "sampled_verify"):
        out, acc, q = model.out_tokens.cpu().numpy(), model.accepted.cpu().numpy(), model.q_len
        return [(b * q + j, int(out[b, j])) for b in range(out.shape[0]) for j in range(int(acc[b]) + 1)]
    if mode == "beam":
        # next beams with a finite cum; a request with fewer finite candidates than W fills its last beams with -inf ones
        # that the ranking by flat index picks from masked tokens: those are exempt
        o, W = model.beam_out, model.W
        tok, par, cum = (o[k].cpu().numpy() for k in ("next_token", "next_parent", "next_cum"))
        return [(b * W + int(par[b, i]), int(tok[b, i])) for b in range(tok.shape[0]) for i in range(W) if np.isfinite(cum[b, i])]
    return list(enumerate(model.next_ids.cpu().numpy().tolist()))


@pytest.mark.parametrize("run", ["eager", "graph pdl"])
@pytest.mark.parametrize("quant", ["int4", "f16"])
@pytest.mark.parametrize("mode", list(MODES))
def test_every_ending_obeys_the_mask_and_the_bias(mode, quant, run):
    model = build(mode, quant, run, keep_reference=True)
    R, V, T = model.B * model.q_len, model.vocab, model.cfg.tokens_per_block
    rng = np.random.default_rng(len(mode) + len(quant) + len(run))
    steps = 6
    seq0 = model.seq_lens_h.clone().long()
    if mode in ("sampling", "beam"):        # these advance one token per step
        assert ((seq0 + steps) // T > seq0 // T).any(), "no page crossing in this run"
    elif mode != "greedy":
        assert ((seq0 + model.q_len - 1) // T > seq0 // T).any(), "no page crossing within a verification step"
    try:
        if "graph" in run:
            model.capture()
        for t in range(steps):
            ok = rng.random((R, V)) < 0.5
            ok[np.arange(R), rng.integers(0, V, R)] = True
            bias = [{int(x): float(rng.normal() * 2) for x in rng.integers(0, V, 5)} if r % 2 else {} for r in range(R)]
            model.set_constraints(pack(ok), bias)
            torch.cuda.synchronize()
            state, kv_before = device_state(model), [bits(L["kv"]) for L in model.layers]
            go(model, run)
            assert np.array_equal(allowed(model.bitmask.cpu().numpy(), V), ok)
            for r, tok in emitted(model, mode):
                assert ok[r, tok], f"step {t}: row {r} emitted masked token {tok}"
            exp = oracle_step(state, kv_before)
            got = model.logits.float().cpu().numpy()
            if model.samp is None:           # greedy, verification and beam constrain the lm_head output in place
                assert np.isneginf(got[~ok]).all(), "masked logits are not -inf"
                for r, m in enumerate(bias):
                    for x, b in m.items():
                        exp[r, x] += b
                check_logits(got, exp, mask=ok)
            else:                            # sampling constrains its fp32 copy; the lm_head output stays raw
                check_logits(got, exp)
                assert (model.samp_logits.cpu().numpy()[~ok] == 0).all(), "a masked token has probability"
    finally:
        ops.set_pdl(False)


# beam search is forced through the mask only: it keeps W beams per request, which one biased token per row cannot fill
FORCING = [(m, h) for m in MODES for h in ("mask", "bias") if (m, h) != ("beam", "bias")]


@pytest.mark.parametrize("mode, how", FORCING, ids=[f"{m}-{h}" for m, h in FORCING])
def test_a_single_allowed_token_or_a_large_bias_forces_it(mode, how):
    model = build(mode)
    R, V = model.B * model.q_len, model.vocab
    rng = np.random.default_rng(11)
    force = np.full(R, int(rng.integers(0, V))) if mode == "beam" else rng.integers(0, V, R)
    if how == "mask":
        ok = np.zeros((R, V), bool)
        ok[np.arange(R), force] = True
        model.set_constraints(pack(ok))
    else:
        model.set_constraints(logit_bias=[{int(x): 1e4} for x in force])
    go(model, "eager")
    if mode == "beam":
        o = model.beam_out
        tok, score = o["cand_token"].cpu().numpy(), o["cand_score"].cpu().numpy()
        assert np.isfinite(score).any() and (tok[np.isfinite(score)] == force[0]).all()
        return
    for r, tok in emitted(model, mode):
        assert tok == force[r], f"row {r}: {tok} instead of the forced {force[r]}"


@pytest.mark.parametrize("mode", ["greedy", "sampling"])
def test_a_toy_grammar_over_graph_replays(mode):
    """The next token must be congruent to 3 * the previous one mod 7: each replay's mask is computed on the host from the
    tokens the previous replay emitted."""
    kw = dict(sampling=SamplingParams(temperature=1.0, min_p=0.05, seed=6), max_new_tokens=10) if mode == "sampling" else {}
    model = DecodeStep(dataclasses.replace(TINY, quant="int4"), 4, 64, DEV, seed=6, pdl=True, token_bitmask=True, **kw)
    if mode == "greedy":                     # the greedy step does not advance: the host feeds each token back
        model.seq_lens_h -= 10
        model.upload_inputs()
    V = model.vocab
    cls = np.arange(V) % 7
    try:
        model.capture()
        prev = model.ids_h.numpy().copy()
        for step in range(8):
            model.set_constraints(pack(cls[None] == (3 * prev[:, None]) % 7))
            model.replay()
            torch.cuda.synchronize()
            tok = model.next_ids.cpu().numpy()
            assert (tok % 7 == (3 * prev) % 7).all(), f"replay {step}: {tok} after {prev}"
            if mode == "greedy":
                model.ids_h.copy_(torch.from_numpy(tok))
                model.seq_lens_h += 1
                model.upload_inputs()
            prev = tok
    finally:
        ops.set_pdl(False)


@pytest.mark.parametrize("mode", ["greedy", "sampling"])
def test_an_all_ones_mask_changes_no_bit(mode):
    cfg = dataclasses.replace(TINY, quant="int4")
    kw = dict(sampling=SamplingParams(top_k=50, seed=2), max_new_tokens=4) if mode == "sampling" else {}
    plain = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=7, pdl=True, **kw)
    cons = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=7, pdl=True, token_bitmask=True, logit_bias_capacity=8, **kw)
    try:
        for m in (plain, cons):
            m.capture()
        cons.set_constraints(np.full(cons.bitmask_h.shape, -1, np.int32), [{}] * cons.B)
        for _ in range(2):
            for m in (plain, cons):
                m.replay()
            torch.cuda.synchronize()
            assert torch.equal(plain.logits.view(torch.int16), cons.logits.view(torch.int16))
            assert torch.equal(plain.next_ids, cons.next_ids)
            if mode == "sampling":
                assert torch.equal(plain.token_prob.view(torch.int32), cons.token_prob.view(torch.int32))
                assert torch.equal(plain.samp_logits.view(torch.int32), cons.samp_logits.view(torch.int32))
    finally:
        ops.set_pdl(False)


def test_constraints_cost_one_launch_and_run_in_a_decode_program():
    cfg = dataclasses.replace(TINY, quant="int4")
    plain = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=7)
    cons = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=7, token_bitmask=True, logit_bias_capacity=8)
    assert cons.launches_per_step() == plain.launches_per_step() + 1
    mask_only = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=7, token_bitmask=True)
    assert mask_only.launches_per_step() == plain.launches_per_step() + 1
    plain.build_program()
    cons.build_program()
    assert cons.prog.num_launches == plain.prog.num_launches + 1
    force = np.array([3, 700, 64, 1023])
    ok = np.zeros((4, cons.vocab), bool)
    ok[np.arange(4), force] = True
    cons.set_constraints(pack(ok))
    n0 = ops.launch_count()
    cons.run()
    torch.cuda.synchronize()
    assert ops.launch_count() - n0 == cons.prog.num_launches
    assert cons.next_ids.cpu().tolist() == force.tolist()
    assert cons.h2d_bytes() == plain.h2d_bytes() + cons.bitmask_h.numel() * 4 + (5 + 8 + 8) * 4
