"""GPU tests (H100) of sampled tree verification with draft rows (b200_spec_verify_tree_draft): the kernel against the float32
restatement of tests/verify_oracle.py at Llama-3's vocabulary, bit for bit with b200_spec_verify(draft_probs) on chains,
the PDL grid dependency and graph replay through the slow-predecessor harness, and DecodeStep(draft_probs=True) for trees and
chains."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams, sampling_uniforms  # noqa: E402
from tests.pdl_cases import I32, Case, Spec  # noqa: E402
from tests.test_gpu_pdl_hazards import _run_case  # noqa: E402
from tests.test_gpu_spec_verify import V_FULL, _probs, check_verify  # noqa: E402
from tests.verify_oracle import chain_verify_np, random_tree, verify_np  # noqa: E402

DEV = torch.device("cuda")


def _T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _sparse(row, keep):
    """row with only its `keep` largest entries, renormalised."""
    out = np.zeros_like(row)
    top = np.argpartition(row, -keep)[-keep:]
    out[top] = row[top]
    return (out / out.astype(np.float64).sum()).astype(np.float32)


def _case(seed, kind, n, B, V=V_FULL):
    """Trees of `kind`, target rows of temperature-0.25 softmaxes (every fifth sparse: 40 tokens), and draft rows of every
    flavour: node c's row is its parent's target row itself (accepted whenever the token has mass), a mix of it with another
    softmax, a sparse row, or a far row; tokens drawn from their rows, with duplicate siblings, and a token outside the
    vocabulary in one sequence."""
    rng = np.random.default_rng(seed)
    par = (np.stack([random_tree(rng, n, kind) for _ in range(B)]) if kind == "random"
           else np.tile(random_tree(rng, n, kind), (B, 1))).astype(np.int32)
    t = _probs(rng, (B, n, V), 0.25)
    other = _probs(rng, (B, n, V), 0.25)
    dp = np.empty((B, n, V), np.float32)
    toks = np.zeros((B, n), np.int32)
    for b in range(B):
        for j in range(n):
            if (b + j) % 5 == 0:
                t[b, j] = _sparse(t[b, j], 40)
        for c in range(1, n):
            parent = t[b, par[b, c]]
            flavour = (b * 7 + c) % 4
            dp[b, c] = (parent if flavour == 0 else (0.5 * parent + 0.5 * other[b, c]).astype(np.float32) if flavour == 1
                        else _sparse(other[b, c], 60) if flavour == 2 else other[b, c])
            row = dp[b, c].astype(np.float64)
            toks[b, c] = rng.choice(V, p=row / row.sum())
    dp[:, 0] = np.nan                                    # row 0 is not read
    toks[:, 0] = -1
    if B > 1:
        kids0 = [c for c in range(1, n) if par[1, c] == 0]
        for c in kids0[1:]:                              # duplicate siblings under sequence 1's root
            toks[1, c] = toks[1, kids0[0]]
    if B > 2:
        toks[2, n - 1] = V + 7                           # outside the vocabulary: rejected
    u = rng.random((B, n)).astype(np.float32)
    return par, toks, t, dp, u


CASES = [("random", 2, 1), ("random", 5, 32), ("random", 16, 8), ("random", 64, 4), ("binary", 8, 32), ("binary", 31, 3),
         ("star", 3, 16), ("star", 12, 8), ("star", 64, 2), ("chain", 4, 32), ("chain", 17, 5)]


@pytest.mark.parametrize("kind,n,B", CASES, ids=[f"{k} n{n} B{B}" for k, n, B in CASES])
def test_tree_draft_verify_vs_fp32_oracle(kind, n, B):
    par, toks, t, dp, u = _case(n * 100 + B, kind, n, B)
    got = ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u), draft_probs=_T(dp))
    exp = verify_np(par, toks, target_probs=t, draft_probs=dp, uniform=u)
    check_verify(got, exp, u[:, n - 1])
    ea = exp[1]
    if n > 2 and B >= 8:
        assert 0 < ea.mean(), "no acceptance"
        assert (ea < n - 1).any(), "no rejection"


def _stop_children(par, ea, ep):
    """How many children the node each sequence's walk stopped at has: all of them were rejected (0: a leaf)."""
    return np.array([(par[b] == ep[b, ea[b]]).sum() for b in range(par.shape[0])])


def test_cases_reach_every_kind_of_stop_node():
    """The draw differs by where the walk stops: at a leaf (from t), after one rejected child (from the residual of one pass
    from t), or after two or more (from the residual the passes rewrote in place). CASES reach all three."""
    kinds = set()
    for kind, n, B in CASES:
        par, toks, t, dp, u = _case(n * 100 + B, kind, n, B)
        _, ea, ep, _ = verify_np(par, toks, target_probs=t, draft_probs=dp, uniform=u)
        kinds |= set(np.minimum(_stop_children(par, ea, ep), 2).tolist())
    assert kinds == {0, 1, 2}, kinds


@pytest.mark.parametrize("V", [1001, 4096])
def test_tree_draft_verify_scalar_pass_vs_fp32_oracle(V):
    """The scalar pass (a vocabulary that is not a multiple of 4, or rows 4 bytes off 16-byte alignment) sums in the order of
    the float4 pass: the oracle's decisions, and with misaligned rows the aligned launch's outputs bit for bit."""
    par, toks, t, dp, u = _case(V, "random", 12, 16, V=V)
    got = ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u), draft_probs=_T(dp))
    check_verify(got, verify_np(par, toks, target_probs=t, draft_probs=dp, uniform=u), u[:, -1])
    if V % 4:
        return
    B, n = par.shape
    flat = torch.empty(1 + t.size, dtype=torch.float32, device=DEV)
    tv = flat[1:].view(B, n, V)                            # 4 bytes past the allocation's alignment
    tv.copy_(_T(t))
    got2 = ops.spec_verify_tree(_T(par), _T(toks), target_probs=tv, uniform=_T(u), draft_probs=_T(dp))
    for a, b in zip(got, got2):
        assert torch.equal(a, b)


@pytest.mark.parametrize("n", [2, 4, 8, 16])
def test_tree_draft_verify_on_a_chain_is_spec_verify_with_draft_probs_bit_for_bit(n):
    par, toks, t, dp, u = _case(7 + n, "chain", n, 32)
    dpt = _T(dp)
    o1, a1 = ops.spec_verify(_T(toks[:, 1:]), target_probs=_T(t), draft_probs=dpt[:, 1:].contiguous(), uniform=_T(u))
    o2, a2, p2 = ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u), draft_probs=dpt)
    assert torch.equal(o1, o2) and torch.equal(a1, a2)
    a = a2.cpu().numpy()
    np.testing.assert_array_equal(p2.cpu().numpy(), [[i if i <= a[b] else -1 for i in range(n)] for b in range(32)])
    assert 0 < a.mean() < n - 1


def test_tree_draft_verify_rejects_with_a_workspace_too_small():
    par, toks, t, dp, u = _case(3, "star", 4, 2, V=500)
    with pytest.raises(ops.B200Error, match="workspace"):
        ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u), draft_probs=_T(dp),
                             workspace=torch.empty(2 * 500 * 4 - 1, dtype=torch.uint8, device=DEV))
    with pytest.raises(ops.B200Error, match="draft_probs must be fp32"):
        ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u), draft_probs=_T(dp[:, 1:]))


# ---------------------------------------------------------------------------------------------------- PDL and graph replay
def _pdl_case(B=4, n=8, V=500):
    def dyn(seed):
        rng = np.random.default_rng(seed)
        par = np.stack([random_tree(rng, n, "random") for _ in range(B)]).astype(np.int32)
        g = torch.Generator().manual_seed(seed)
        return dict(par=_T(par), tok=torch.randint(0, V, (B, n), generator=g, dtype=I32).to(DEV),
                    tp=torch.softmax(torch.randn(B, n, V, generator=g) * 2, -1).to(DEV),
                    dp=torch.softmax(torch.randn(B, n, V, generator=g) * 2, -1).to(DEV),
                    u=torch.rand(B, n, generator=g).to(DEV))

    def call(b):
        ops.spec_verify_tree(b["par"], b["tok"], target_probs=b["tp"], uniform=b["u"], draft_probs=b["dp"], workspace=b["ws"],
                             out_tokens=b["o"], accepted=b["a"], accepted_path=b["p"])

    def setup():
        return Spec(dyn, call, outs=dict(o=((B, n), I32), a=((B,), I32), p=((B, n), I32)), ws=dict(ws=(B * V * 4, 0)))
    return Case("spec_verify_tree draft rows", ("spec_verify_kernel",), setup)


def test_tree_draft_verify_waits_for_its_grid_dependency():
    """The slow-predecessor harness: under PDL, in a stream and replayed from a CUDA graph on three staged inputs, every output
    and the residual workspace hold the bits of a plain launch on the inputs the predecessor left."""
    _run_case(_pdl_case())


# ---------------------------------------------------------------------------------------------------- decode step
def _run(model, mode):
    try:
        if "graph" in mode:
            model.replay()
        else:
            model.run()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)


TREE = [-1, 0, 0, 1, 1, 2, 3]                   # first-child path 0, 1, 3, 6: depth 3


@pytest.mark.parametrize("mode", ["eager", "graph", "graph pdl"])
def test_tree_step_with_its_own_rows_as_draft_rows_accepts_every_first_child(mode):
    """Run the step, set each node's draft row to its parent's target row and run the same inputs again: every first child is
    accepted (u * q(x) * 1 < q(x) for q(x) > 0; no top-k / top-p, so every token has mass), so accepted is the depth of the
    first-child path; the logits and the target rows are those of the same step without draft rows, bit for bit; and the
    decisions are the fp32 oracle's on the step's own rows and uniforms."""
    cfg = dataclasses.replace(TINY, quant="int4")
    sp = SamplingParams(temperature=0.9, seed=7)
    n, kw = len(TREE), dict(ragged=True, seed=3, q_len=len(TREE), tree=TREE, sampling=sp, pdl="pdl" in mode)
    plain = DecodeStep(cfg, 4, 40, DEV, **kw)
    m = DecodeStep(cfg, 4, 40, DEV, draft_probs=True, **kw)
    B, R = m.B, m.B * n
    if "graph" in mode:                         # (both captured while the constructors' PDL setting holds)
        plain.capture()
        m.capture()
    _run(plain, mode)
    _run(m, mode)
    tp = m.target_probs.clone()
    par = torch.tensor(TREE, device=DEV).clamp(min=0)
    m.set_draft_probs(tp[:, par].contiguous())
    m.upload_inputs()
    _run(m, mode)
    assert torch.equal(m.logits.view(torch.int16), plain.logits.view(torch.int16)), "logits differ"
    assert torch.equal(m.target_probs, plain.target_probs) and torch.equal(m.target_probs, tp)
    acc, path = m.accepted.cpu().numpy(), m.accepted_path.cpu().numpy()
    assert (acc == 3).all(), acc
    assert (path == [0, 1, 3, 6, -1, -1, -1]).all(), path
    u = sampling_uniforms(sp.seed, 0, 2 * R)[R:].view(B, n).numpy()
    assert torch.equal(m.uniform[R:].cpu(), torch.from_numpy(u).view(-1))
    toks = m.ids_h.numpy()
    got = (m.out_tokens, m.accepted, m.accepted_path)
    exp = verify_np(np.tile(TREE, (B, 1)), toks, target_probs=tp.cpu().numpy(), draft_probs=m.draft_probs.cpu().numpy(),
                    uniform=u)
    check_verify(got, exp, u[:, n - 1])


@pytest.mark.parametrize("mode", ["eager", "graph pdl"])
def test_chain_step_with_draft_rows_vs_oracle(mode):
    """The chain verification step with draft rows (a mix of the step's own target rows and a far distribution): out_tokens and
    accepted are chain_verify_np's on the step's own target_probs, draft_probs and uniforms, for several drafts."""
    cfg = dataclasses.replace(TINY, quant="int4")
    sp = SamplingParams(temperature=[0.7, 1.0, 1.3, 1.0], top_k=[0, 50, 0, 20], top_p=[1.0, 0.9, 0.95, 1.0], seed=11)
    q_len = 4
    m = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=5, q_len=q_len, sampling=sp, draft_probs=True, pdl="pdl" in mode)
    B, R = m.B, m.B * q_len
    g = torch.Generator().manual_seed(1)
    if "graph" in mode:
        m.capture()
    _run(m, mode)
    far = torch.softmax(torch.randn(B, q_len - 1, m.vocab, generator=g) * 3, -1)
    accepted = []
    for w in (1.0, 0.6, 0.0):
        m.set_draft_probs((w * m.target_probs[:, :q_len - 1].cpu() + (1 - w) * far).contiguous())
        m.upload_inputs()
        _run(m, mode)
        tp, dp = m.target_probs.cpu().numpy(), m.draft_probs.cpu().numpy()
        u = sampling_uniforms(sp.seed, 0, 2 * R)[R:].view(B, q_len).numpy()
        eo, ea = chain_verify_np(m.ids_h[:, 1:].numpy(), target_probs=tp, draft_probs=dp, uniform=u)[:2]
        np.testing.assert_array_equal(m.accepted.cpu().numpy(), ea)
        np.testing.assert_array_equal(m.out_tokens.cpu().numpy(), eo)
        accepted.append(ea.mean())
    assert accepted[0] >= accepted[-1]
