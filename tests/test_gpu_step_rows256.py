"""GPU tests (H100): every decode-step mode at its 256-row shape, where each GEMM of the step runs the batch-pad-256 instance
of the weight-only GEMM (129..256 token rows).

The verification, tree, beam and sampling modes run with max_rows=256 (their default stays 128 rows).

- Against the whole-step oracle (tests/step_oracle.py, its one tolerance): greedy at B 256 (TINY int4 / f16, TINY_QWEN3),
  verification at B 64 x q_len 4 with the verifier's decisions, the shared-prefix step at B 256 in groups of 8; eagerly and
  captured in a CUDA graph with PDL.
- Graph + PDL against eager, bit for bit over 6 steps on changing inputs (test_gpu_pdl_steps' harness): greedy, verification,
  a binary / random tree at B 32 x 8 nodes, beam at B 64 x W 4 with eos_id, sampling at B 256 with penalties and log-probs,
  constrained greedy, QK-norm and act-order at B 256.
- A decode program at B 200 gives the logits and K/V pools of the same step run op by op, bit for bit."""
import dataclasses
import functools

import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, TINY_QWEN3, DecodeStep, SamplingParams  # noqa: E402
from tests import step_oracle  # noqa: E402
from tests import test_gpu_pdl_steps as ps  # noqa: E402
from tests.step_oracle import bits, check_logits, check_step, oracle_step  # noqa: E402

DEV = torch.device("cuda")
INT4 = dataclasses.replace(TINY, quant="int4")
SAMPLING = SamplingParams(temperature=0.9, top_k=50, top_p=0.9, repetition=1.2, presence=0.5, frequency=0.1, seed=11)


@pytest.mark.parametrize("mode", ["eager", "graph pdl"])
@pytest.mark.parametrize("cfg,quant,batch,q_len", [(TINY, "int4", 256, 1), (TINY, "f16", 256, 1), (TINY_QWEN3, "int4", 256, 1),
                                                   (TINY, "int4", 64, 4)],
                         ids=["greedy int4 B256", "greedy f16 B256", "qwen3 B256", "verify B64 x q_len 4"])
def test_step_against_the_oracle_at_256_rows(cfg, quant, batch, q_len, mode, monkeypatch):
    monkeypatch.setattr(step_oracle, "DecodeStep", functools.partial(DecodeStep, max_rows=256))
    check_step(cfg, quant=quant, batch=batch, q_len=q_len, mode=mode)


@pytest.mark.parametrize("mode", ["eager", "graph pdl"])
def test_shared_prefix_step_at_256_rows(mode):
    model = DecodeStep(INT4, 256, 100, DEV, keep_reference=True, ragged=True, seed=2, pdl="pdl" in mode, shared_prefix=(8, 48))
    try:
        kv_before = [bits(L["kv"]) for L in model.layers]
        if "graph" in mode:
            model.capture()
            model.replay()
        else:
            model.run()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)
    check_logits(model.logits.float().cpu().numpy(), oracle_step(model, kv_before))


# name: (config, DecodeStep keywords, decode program, BATCH of test_gpu_pdl_steps: requests, halved for beam search)
MODES = {
    "greedy int4 B256": (INT4, {}, False, 256),
    "verify B64 x q_len 4": (INT4, dict(q_len=4, max_rows=256), False, 64),
    "tree B32 x 8 nodes": (INT4, dict(q_len=8, tree=[-1, 0, 0, 1, 1, 2, 2, 3], max_rows=256), False, 32),
    "beam B64 x W4 eos": (INT4, dict(beam_width=4, max_new_tokens=8, max_rows=256), False, 128),
    "sampling B256 penalties logprobs": (INT4, dict(sampling=SAMPLING, logprobs=5, max_new_tokens=8, max_rows=256), False, 256),
    "constrained greedy B256": (INT4, dict(token_bitmask=True, logit_bias_capacity=1024), False, 256),
    "qwen3 qk-norm B256": (dataclasses.replace(TINY_QWEN3, quant="int4"), {}, False, 256),
    "act-order B256": (INT4, dict(act_order=True), False, 256),
}


@pytest.mark.parametrize("name", list(MODES))
def test_graph_pdl_steps_equal_eager_steps_at_256_rows(name, monkeypatch):
    cfg, kw, program, batch = MODES[name]
    monkeypatch.setattr(ps, "MODES", {name: (cfg, kw, program)})
    monkeypatch.setattr(ps, "BATCH", batch)
    monkeypatch.setattr(ps, "SEQ0", ps.SEQ0.repeat(batch // 4))
    ps.test_graph_pdl_steps_equal_eager_steps_on_changing_inputs(name)


def test_decode_program_at_200_rows_is_the_op_by_op_step():
    """The GEMMs at batch pad 256 are launches of their own inside the program; the glue ops stay the persistent kernel's."""
    models = [DecodeStep(INT4, 200, 40, DEV, ragged=True, seed=6) for _ in range(2)]
    models[0].build_program()
    for m in models:
        m.run()
    torch.cuda.synchronize()
    got, exp = models
    assert torch.equal(got.logits.view(torch.int16), exp.logits.view(torch.int16))
    for a, b in zip(got.layers, exp.layers):
        assert torch.equal(a["kv"].view(torch.int16), b["kv"].view(torch.int16))
