import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.step_oracle import check_step  # noqa: E402


@pytest.mark.parametrize("quant", ["int4", "int8", "int8g", "f16"])
def test_tiny_decode_step_matches_oracle(quant):
    check_step(quant=quant, batch=3, ctx=40)


def test_tiny_decode_step_under_cuda_graph():
    check_step(quant="int4", batch=5, ctx=70, mode="graph")


def test_tiny_decode_step_with_programmatic_dependent_launch():
    check_step(quant="int4", batch=5, ctx=70, mode="graph+pdl")
    check_step(quant="int8", batch=3, ctx=40, mode="pdl")


@pytest.mark.parametrize("quant", ["int4", "int8", "f16"])
def test_tiny_decode_step_as_program(quant):
    """The same step recorded into a decode program (GEMMs / norms / rope fused into the persistent kernel)."""
    check_step(quant=quant, batch=3, ctx=40, mode="program")


def test_tiny_decode_step_as_program_under_cuda_graph_with_pdl():
    check_step(quant="int4", batch=5, ctx=70, mode="program+graph+pdl")
    check_step(quant="int8", batch=17, ctx=70, mode="program+graph")


def test_program_replays_are_identical_and_match_op_by_op():
    """A program replay must give the same logits every time (fixed summation orders) and agree with the op-by-op step
    within a tolerance: op by op, the GEMMs run in the cluster kernel, whose split-K plan and merge order differ from the
    persistent kernel's, and the norm reduces in a different order."""
    import dataclasses
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    dev = torch.device("cuda:0")
    cfg = dataclasses.replace(TINY, quant="int4", layers=3)
    m = DecodeStep(cfg, 9, 100, dev, ragged=True, seed=3)
    m.step()
    torch.cuda.synchronize()
    ref = m.logits.clone()
    m.build_program()
    outs = []
    for _ in range(3):
        m.run()
        torch.cuda.synchronize()
        outs.append(m.logits.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    scale = ref.float().pow(2).mean().sqrt().item()
    assert (outs[0].float() - ref.float()).abs().max().item() <= 2e-2 * scale + 2e-2
    assert m.prog.num_launches < m.prog.num_ops


def test_tiny_decode_step_with_rope_fused_into_attention():
    check_step(quant="int4", batch=5, ctx=70, mode="graph+pdl", fuse_rope=True)
    check_step(quant="int8", batch=3, ctx=40, mode="program", fuse_rope=True)
