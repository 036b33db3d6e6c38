"""GPU tests (H100) of Qwen3 decoder layers in DecodeStep (ModelConfig.qk_norm): the tiny QK-norm config against the step
oracle in every mode (eager, CUDA graph + PDL, decode program, verification steps, act-order, Qwen3's YaRN), sampling and beam
modes, the step's logits bit for bit against a two-launch composition (qk_rmsnorm, then the plain rope launch), and the
launch count of a QK-norm step."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops, rope  # noqa: E402
from rtp_llm_b200.decode_step import TINY_QWEN3, DecodeStep, SamplingParams, sampling_uniforms  # noqa: E402
from tests.beam_oracle import beam_step_np, check_beam  # noqa: E402
from tests.step_oracle import TwoLaunchStep, bits, check_logits, check_step, device_state, oracle_step  # noqa: E402

DEV = torch.device("cuda")
# Qwen3's YaRN (rope_scaling factor 4, beta_fast 32, beta_slow 1, mscale 0.1 ln 4 + 1) with original max positions 16, so the
# tiny contexts (positions 20..70) sit in the scaled band and the cos/sin table covers them
YARN = rope.RopeSpec(style=rope.YARN, dim=128, base=1000000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=16, mscale=1.1386)
TINY_QWEN3_YARN = dataclasses.replace(TINY_QWEN3, rope=YARN)


@pytest.mark.parametrize("quant", ["int4", "f16", "int8", "int8g"])
@pytest.mark.parametrize("mode", ["eager", "graph pdl", "program"])
def test_qwen3_step_vs_oracle(quant, mode):
    check_step(TINY_QWEN3, quant=quant, batch=3, ctx=40, mode=mode, dev=DEV)


@pytest.mark.parametrize("q_len", [2, 4])
@pytest.mark.parametrize("mode", ["eager", "graph pdl"])
def test_qwen3_verification_step_vs_oracle(q_len, mode):
    check_step(TINY_QWEN3, quant="int4", batch=3, ctx=40, mode=mode, q_len=q_len, dev=DEV)


@pytest.mark.parametrize("quant", ["int4", "int8g"])
def test_qwen3_act_order_step_vs_oracle(quant):
    check_step(TINY_QWEN3, quant=quant, batch=3, ctx=40, mode="graph pdl", act_order=True, dev=DEV)


@pytest.mark.parametrize("case", [(1, "eager"), (1, "program graph pdl"), (4, "graph pdl")])
def test_qwen3_yarn_step_vs_oracle(case):
    q_len, mode = case
    check_step(TINY_QWEN3_YARN, quant="int4", batch=3, ctx=40, mode=mode, q_len=q_len, dev=DEV)


def _pair(cfg, **kw):
    return DecodeStep(cfg, 3, 40, DEV, ragged=True, seed=5, **kw), TwoLaunchStep(cfg, 3, 40, DEV, ragged=True, seed=5, **kw)


@pytest.mark.parametrize("cfg", [TINY_QWEN3, TINY_QWEN3_YARN], ids=["base", "yarn"])
@pytest.mark.parametrize("q_len", [1, 4])
def test_logits_equal_the_two_launch_composition(cfg, q_len):
    fused, two = _pair(dataclasses.replace(cfg, quant="int4"), q_len=q_len, pdl=True)
    try:
        for m in (fused, two):
            m.capture()
            m.replay()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)
    assert torch.equal(fused.logits, two.logits)
    assert all(torch.equal(a["kv"], b["kv"]) for a, b in zip(fused.layers, two.layers))


def test_launches_per_step_equal_those_without_qk_norm():
    """Eager / graph: the fused launch replaces the rope launch. In a program the plain Base rope is an op of the persistent
    kernel while the QK-norm append is its own launch, so there a non-Base config (its rope also its own launch) is the match."""
    cfg = dataclasses.replace(TINY_QWEN3, quant="int4")
    plain = dataclasses.replace(cfg, qk_norm=False)
    n = {c.qk_norm: DecodeStep(c, 3, 40, DEV, ragged=True).launches_per_step() for c in (cfg, plain)}
    assert n[True] == n[False]
    two = TwoLaunchStep(cfg, 3, 40, DEV, ragged=True).launches_per_step()
    assert two == n[True] + cfg.layers
    progs = {}
    for c in (dataclasses.replace(TINY_QWEN3_YARN, quant="int4"), dataclasses.replace(TINY_QWEN3_YARN, quant="int4", qk_norm=False)):
        m = DecodeStep(c, 3, 40, DEV, ragged=True)
        m.build_program()
        progs[c.qk_norm] = m.launches_per_step()
    assert progs[True] == progs[False]


def test_qwen3_sampling_steps():
    """Three sampled steps under a CUDA graph with PDL: every step's logits against the oracle, the same logits, tokens and state
    as the two-launch composition, and the greedy (top_k 1) request's token the argmax of the logits."""
    sp = SamplingParams(temperature=[0.7, 1.0, 1.2], top_k=[1, 50, 0], top_p=[1.0, 0.9, 0.8], seed=13)
    kw = dict(keep_reference=True, sampling=sp, max_new_tokens=8, pdl=True)
    fused, two = _pair(dataclasses.replace(TINY_QWEN3, quant="int4"), **kw)
    try:
        for m in (fused, two):
            m.capture()
        for t in range(3):
            torch.cuda.synchronize()
            state, kv_before = device_state(fused), [bits(L["kv"]) for L in fused.layers]
            for m in (fused, two):
                m.replay()
            torch.cuda.synchronize()
            check_logits(fused.logits.float().cpu().numpy(), oracle_step(state, kv_before))
            assert torch.equal(fused.logits, two.logits) and torch.equal(fused.next_ids, two.next_ids)
            assert torch.equal(fused.uniform.cpu(), sampling_uniforms(sp.seed, t, fused.B))
            assert int(fused.next_ids[0]) == int(fused.logits[0].float().argmax())
            n = int(fused.hist_len.max())                  # the history rows are only written up to hist_len
            assert torch.equal(fused.hist_len, two.hist_len) and torch.equal(fused.hist[:, :n], two.hist[:, :n])
            assert torch.equal(fused.seq_lens, two.seq_lens)
    finally:
        ops.set_pdl(False)


def test_qwen3_beam_steps():
    """Three beam-search steps (width 4) op by op: every step's logits against the oracle on the forked state, the selection
    against the float64 reference, and logits, selections and fork bit for bit equal to the two-launch composition."""
    fused = DecodeStep(dataclasses.replace(TINY_QWEN3, quant="int4"), 2, 40, DEV, keep_reference=True, ragged=True, seed=6,
                       beam_width=4)
    two = TwoLaunchStep(fused.cfg, 2, 40, DEV, keep_reference=True, ragged=True, seed=6, beam_width=4)
    for t in range(3):
        torch.cuda.synchronize()
        state, kv_before = device_state(fused), [bits(L["kv"]) for L in fused.layers]
        cum = fused.beam_cum.cpu().numpy()
        for m in (fused, two):
            m.run()
        torch.cuda.synchronize()
        got = fused.logits.float().cpu().numpy()
        check_logits(got, oracle_step(state, kv_before))
        sel = {k: v.cpu() for k, v in fused.beam_out.items()}
        check_beam({k: v.numpy() for k, v in sel.items()}, beam_step_np(got, cum), 4, -1)
        assert torch.equal(fused.logits, two.logits)
        assert all(torch.equal(sel[k], v.cpu()) for k, v in two.beam_out.items())
        n = int(fused.hist_len.max())
        assert torch.equal(fused.block_ids, two.block_ids) and torch.equal(fused.hist[:, :n], two.hist[:, :n])
        assert all(torch.equal(a["kv"], b["kv"]) for a, b in zip(fused.layers, two.layers))
