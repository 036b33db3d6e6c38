"""GPU tests (H100): decode steps captured under a CUDA graph with programmatic dependent launch (PDL) give the bits of the same
steps run eagerly with PDL off, step after step, on inputs that change between steps.

A graph replayed on the inputs of its warm-up runs cannot show a stale read: the bits a kernel would read before its
griddepcontrol.wait are the ones the warm-up left, which are the right ones. Here two DecodeSteps of one seed run 6 steps
each; before every step the greedy, verification, tree and constrained steps take new token ids and lengths (crossing page
boundaries), new trees and new masks and bias, and the beam and sampling steps advance on the device by themselves. After each
step the logits, the ending's outputs and every layer's whole K/V pool must be equal bit for bit. PDL is switched library-wide,
so the test sets it explicitly before each model's work."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, TINY_QWEN3, DecodeStep  # noqa: E402
from tests.test_gpu_sampling import PARAMS  # noqa: E402
from tests.verify_oracle import random_tree  # noqa: E402

DEV = torch.device("cuda")
STEPS, BATCH, CTX = 6, 4, 40
SEQ0 = torch.tensor([13, 29, 30, 10], dtype=torch.int32)   # + 0..5 crosses the page boundaries at 16 and 32 (16 tokens a page)
INT4 = dataclasses.replace(TINY, quant="int4")

MODES = {   # name: (config, DecodeStep keywords, built as a decode program)
    "greedy int4": (INT4, {}, False),
    "greedy f16": (dataclasses.replace(TINY, quant="f16"), {}, False),
    "verify q_len 4": (INT4, dict(q_len=4), False),
    "tree binary / random": (INT4, dict(q_len=5, tree=[-1, 0, 0, 1, 1]), False),
    "beam w4 eos": (INT4, dict(beam_width=4, max_new_tokens=8), False),
    "sampling penalties logprobs": (INT4, dict(sampling=PARAMS, logprobs=5, max_new_tokens=8), False),
    "constrained greedy": (INT4, dict(token_bitmask=True, logit_bias_capacity=64), False),
    "qwen3 qk-norm": (dataclasses.replace(TINY_QWEN3, quant="int4"), {}, False),
    "act-order": (INT4, dict(act_order=True), False),
    "program": (INT4, {}, True),
}


def _eos(cfg, kw) -> int:
    """A token among the first W candidates of a first beam step, so that finished hypotheses do occur."""
    m = DecodeStep(cfg, BATCH // 2, CTX, DEV, ragged=True, seed=5, **kw)
    m.run()
    torch.cuda.synchronize()
    return int(m.beam_out["cand_token"][0, 1])


def _build(cfg, kw, program, pdl):
    ops.set_pdl(pdl)
    batch = BATCH // 2 if kw.get("beam_width", 1) > 1 else BATCH
    m = DecodeStep(cfg, batch, CTX, DEV, ragged=True, seed=5, pdl=pdl, **kw)
    if program:
        m.build_program()
    return m


def _warm(m):
    """What capture() runs before it records the step, for the eager twin: the same K/V appends and state."""
    advances = m.W > 1 or m.samp is not None
    for _ in range(2):
        m.run()
        if advances:
            m.upload_inputs()
    if advances:
        m.upload_inputs()


def _feed(m, k):
    """New inputs of step k for a step that does not advance by itself: ids, lengths, tree, constraints."""
    if m.W > 1 or m.samp is not None:
        return
    g = torch.Generator().manual_seed(100 + k)
    m.ids_h.copy_(torch.randint(0, m.vocab, tuple(m.ids_h.shape), generator=g, dtype=torch.int32))
    m.seq_lens_h.copy_(SEQ0 + k)
    m.upload_inputs()
    if m.tree_parents is not None:
        rng = np.random.default_rng(k)
        m.set_tree([[int(p) for p in random_tree(rng, m.q_len, "binary" if k % 2 else "random")] for _ in range(m.B)])
    if m.bitmask is not None:
        R, words = m.bitmask_h.shape
        mask = torch.randint(-2 ** 31, 2 ** 31 - 1, (R, words), generator=g, dtype=torch.int32)
        mask |= torch.randint(-2 ** 31, 2 ** 31 - 1, (R, words), generator=g, dtype=torch.int32)    # 3 in 4 tokens allowed
        bias = [{int(t): float(v) for t, v in zip(torch.randperm(m.vocab, generator=g)[:4], torch.randn(4, generator=g) * 3)}
                for _ in range(R)]
        m.set_constraints(mask, bias)


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8)


def _state(m) -> dict:
    s = {"logits": m.logits}
    if m.W == 1:                       # the beam ending's tokens are beam_out's; next_ids is not written there
        s["next_ids"] = m.next_ids
    for k in ("out_tokens", "accepted", "accepted_path", "hyp_state", "done", "beam_cum", "cum_log_probs", "hist_len", "ids",
              "seq_lens"):
        if isinstance(getattr(m, k, None), torch.Tensor):
            s[k] = getattr(m, k)
    if m.advances:                     # the token history up to each row's length (the rest of the buffer is never written)
        live = torch.arange(m.hist.shape[1], device=m.hist.device).view(1, -1) < m.hist_len.view(-1, 1)
        s["hist"] = torch.where(live, m.hist, torch.zeros_like(m.hist))
    for group in ("beam_out", "lp_out"):
        for k, v in (getattr(m, group, None) or {}).items():
            s[f"{group}.{k}"] = v
    for i, L in enumerate(m.layers):
        s[f"kv{i}"] = L["kv"]
    return {k: v.detach().clone() for k, v in s.items()}


@pytest.mark.parametrize("name", list(MODES))
def test_graph_pdl_steps_equal_eager_steps_on_changing_inputs(name):
    cfg, kw, program = MODES[name]
    if "beam_width" in kw:
        kw = dict(kw, eos_id=_eos(cfg, kw))
    try:
        graphed = _build(cfg, kw, program, pdl=True)
        graphed.capture()
        eager = _build(cfg, kw, program, pdl=False)
        _warm(eager)
        torch.cuda.synchronize()
        assert torch.equal(graphed.seq_lens, eager.seq_lens)
        for k in range(STEPS):
            ops.set_pdl(True)
            _feed(graphed, k)
            graphed.replay()
            ops.set_pdl(False)
            _feed(eager, k)
            eager.run()
            torch.cuda.synchronize()
            got, exp = _state(graphed), _state(eager)
            assert got.keys() == exp.keys()
            bad = [f"{key} ({int((_bytes(got[key]) != _bytes(exp[key])).sum())} bytes)"
                   for key in exp if not torch.equal(_bytes(got[key]), _bytes(exp[key]))]
            assert not bad, f"{name} step {k}: graph + PDL differs from eager in " + ", ".join(bad)
        if not (kw.get("beam_width", 1) > 1 or "sampling" in kw):
            T = cfg.tokens_per_block
            assert (((SEQ0 + STEPS - 1) // T) > (SEQ0 // T)).any(), "no page crossing in this run"
    finally:
        ops.set_pdl(False)
