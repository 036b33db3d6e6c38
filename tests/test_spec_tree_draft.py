"""CPU tests of sampled tree verification with draft rows (b200_spec_verify_tree_draft): the rule of tests/verify_oracle.py
emits the target's distribution exactly (SpecInfer's theorem, in float64 over every draft and uniform) and is the deterministic-
draft rule with one-hot rows; and the host checks of the C entry, of ops and of DecodeStep's draft_probs option."""
import ctypes

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams
from tests.verify_oracle import block_sum_f32, exact_emitted, extend, random_tree, target_joint, verify_measure, verify_np


def _row(key, V, zeros):
    """A float64 distribution over V tokens that is a function of `key` (an int tuple), with about `zeros` of its entries 0."""
    rng = np.random.default_rng(abs(hash(key)) % (1 << 32))
    r = rng.random(V) ** 2 + 0.05
    r[rng.random(V) < zeros] = 0.0
    if r.sum() == 0:
        r[rng.integers(0, V)] = 1.0
    return r / r.sum()


def _depth(parents):
    d = [0] * len(parents)
    for c in range(1, len(parents)):
        d[c] = d[parents[c]] + 1
    return max(d)


TREES = {"star 3": [-1, 0, 0, 0], "binary 6": [-1, 0, 0, 1, 1, 2], "chain 4": [-1, 0, 1, 2], "random 6": [-1, 0, 0, 1, 2, 2],
         "wide and deep 5": [-1, 0, 0, 2, 2]}


@pytest.mark.parametrize("without_replacement", [False, True], ids=["iid siblings", "siblings without replacement"])
@pytest.mark.parametrize("drafter", ["mixed", "far", "equal"])
@pytest.mark.parametrize("name", list(TREES))
def test_recursive_rejection_emits_the_target_distribution(name, drafter, without_replacement):
    """Over every draft of the tree (drawn from the drafter's rows) and every uniform, the emitted tokens continued by the target
    to depth + 1 tokens have the target's own measure, to 1e-12: the rule is unbiased, whatever the drafter and however the
    siblings repeat (target rows are a function of the token path, so duplicate siblings share their subtree's rows)."""
    par = TREES[name]
    V = 3 if len(par) > 5 else 4
    seed = sum(map(ord, name))
    z = 0.0 if without_replacement else 0.3       # (siblings drawn without replacement need as many tokens with mass)
    target = lambda path: _row((seed, 1) + path, V, z)
    draft = {"mixed": lambda path: 0.5 * target(path) + 0.5 * _row((seed, 2) + path, V, z),
             "far": lambda path: _row((seed, 3) + path, V, 1.5 * z),
             "equal": target}[drafter]
    L = _depth(par) + 1
    got = extend(exact_emitted(par, draft, target, V, without_replacement=without_replacement), target, L)
    exp = target_joint(target, V, L)
    assert abs(sum(got.values()) - 1.0) < 1e-12
    keys = set(got) | set(exp)
    err = max(abs(got.get(k, 0.0) - exp.get(k, 0.0)) for k in keys)
    assert err < 1e-12, (name, drafter, err)


def test_a_drafter_equal_to_the_target_accepts_the_whole_path():
    """p = q at every node: every first child is accepted (min(1, q / q) = 1), so the emitted path is as deep as the tree."""
    par = TREES["binary 6"]
    target = lambda path: _row((9,) + path, 3, 0.2)
    toks = (-1, 0, 1, 2, 0, 1)
    paths = [()]
    for c in range(1, len(par)):
        paths.append(paths[par[c]] + (toks[c],))
    rows = [None] + [target(paths[par[c]]) for c in range(1, len(par))]
    if any(rows[c][toks[c]] == 0 for c in (1, 3)):
        pytest.skip("a first-child token without target mass")
    m = verify_measure(par, toks, rows, target)
    assert abs(sum(p for s, p in m.items() if s[:2] == (toks[1], toks[3])) - 1.0) < 1e-12


@pytest.mark.parametrize("name", list(TREES))
def test_one_hot_rows_are_the_deterministic_draft_rule(name):
    """Draft rows one-hot at each node's token: the measure of the emitted tokens is b200_spec_verify_tree's (multi-round
    rejection of deterministic drafts), exactly, for every drafted tree including repeated sibling tokens."""
    par = TREES[name]
    V = 3
    target = lambda path: _row((5,) + path, V, 0.3)
    rng = np.random.default_rng(len(par))
    for _ in range(12):
        toks = (-1,) + tuple(int(x) for x in rng.integers(0, V, len(par) - 1))
        rows = [None] + [np.eye(V)[toks[c]] for c in range(1, len(par))]
        got = verify_measure(par, toks, rows, target, "draft")
        exp = verify_measure(par, toks, rows, target, "deterministic")
        keys = set(got) | set(exp)
        assert max(abs(got.get(k, 0.0) - exp.get(k, 0.0)) for k in keys) < 1e-12, toks


def _probs(rng, shape, temp, zeros=0.0):
    x = rng.standard_normal(shape) / temp
    p = np.exp(x - x.max(-1, keepdims=True))
    p[rng.random(shape) < zeros] = 0.0
    return (p / np.maximum(p.sum(-1, keepdims=True), 1e-30)).astype(np.float32)


@pytest.mark.parametrize("seed", range(4))
def test_fp32_oracle_with_one_hot_rows_decides_as_the_deterministic_oracle(seed):
    rng = np.random.default_rng(seed)
    B, n, V = 48, int(rng.integers(3, 10)), 40
    par = np.stack([random_tree(rng, n, rng.choice(["random", "star", "binary"])) for _ in range(B)])
    t = _probs(rng, (B, n, V), 0.5, zeros=0.2)
    toks = rng.integers(0, V, (B, n))
    toks[:, 0] = -3
    toks[0, 1:] = toks[0, 1]                                                 # duplicate siblings
    dp = np.zeros((B, n, V), np.float32)
    for b in range(B):
        for c in range(1, n):
            dp[b, c, toks[b, c]] = 1.0
    u = rng.random((B, n)).astype(np.float32)
    got = verify_np(par, toks, target_probs=t, draft_probs=dp, uniform=u)
    exp = verify_np(par, toks, target_probs=t, uniform=u)
    for g, e in zip(got[:3], exp[:3]):
        np.testing.assert_array_equal(g, e)
    assert 0 < got[1].mean()


def test_block_sum_order():
    """The kernel's order on values whose sum is exact, and a case where the order decides the last bit."""
    r = np.arange(5000, dtype=np.float32)
    assert block_sum_f32(r) == np.float32(r.astype(np.float64).sum())
    x = np.zeros(4100, np.float32)
    x[0], x[1], x[4096] = 1.0, 2.0 ** -24, 2.0 ** -24      # thread 0: (1 + 2^-24) + 2^-24 rounds twice; the exact sum does not
    assert block_sum_f32(x) == np.float32(1.0)
    assert np.float32(x.astype(np.float64).sum()) != np.float32(1.0)


# ---------------------------------------------------------------------------------------------------- host checks
@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_workspace_bytes(lib):
    assert lib.b200_spec_verify_tree_draft_workspace_bytes(4, 100) == 1600
    assert lib.b200_spec_verify_tree_draft_workspace_bytes(32, 128256) == 32 * 128256 * 4
    assert lib.b200_spec_verify_tree_draft_workspace_bytes(0, 100) == 0


def test_entry_argument_checks(lib):
    buf = (ctypes.c_uint8 * (1 << 16))()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = lib.b200_spec_verify_tree_draft

    def call(batch=2, n=4, vocab=100, ws_bytes=800, ptrs=None):
        a = ptrs or [p] * 9       # target, draft, parents, tokens, uniform, workspace, out_tokens, accepted, path
        return f(a[0], a[1], a[2], a[3], a[4], batch, n, vocab, a[5], ws_bytes, a[6], a[7], a[8], None)

    def err():
        return lib.b200_last_error()
    assert call(n=1) == -1 and b"n 1" in err() and b"2..64" in err() and b"spec_verify_tree_draft" in err()
    assert call(n=65) == -1 and b"2..64" in err()
    assert call(vocab=0) == -1 and b"vocab" in err()
    assert call(batch=70000) == -1 and b"batch" in err()
    assert call(batch=-1) == -1 and b"batch" in err()
    for i in range(9):
        a = [p] * 9
        a[i] = None
        assert call(ptrs=a) == -1, i
        assert (b"workspace" if i == 5 else b"null") in err(), i
    assert call(ws_bytes=799) == -1 and b"workspace too small" in err() and b"799 < 800" in err()
    assert f(None, None, None, None, None, 0, 4, 100, None, 0, None, None, None, None) == 0     # empty batch: no work


def test_ops_rejects_draft_probs_in_greedy_mode():
    par = torch.zeros(2, 4, dtype=torch.int32)
    with pytest.raises(_lib.B200Error, match="draft_probs need the sampling mode"):
        ops.spec_verify_tree(par, par, target_ids=par, draft_probs=torch.zeros(2, 4, 8))


def test_decode_step_draft_probs_option_checks():
    samp = SamplingParams(temperature=0.8, top_k=50, seed=1)
    with pytest.raises(ValueError, match="draft_probs needs sampled verification"):
        DecodeStep(TINY, 4, 40, None, q_len=4, draft_probs=True)                        # greedy verification
    with pytest.raises(ValueError, match="draft_probs needs sampled verification"):
        DecodeStep(TINY, 4, 40, None, q_len=4, tree=[-1, 0, 0, 1], draft_probs=True)    # greedy tree
    with pytest.raises(ValueError, match="draft_probs needs sampled verification"):
        DecodeStep(TINY, 4, 40, None, sampling=samp, draft_probs=True)                   # q_len 1: nothing to verify
    with pytest.raises(ValueError, match="draft_probs needs sampled verification"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, draft_probs=True)
    # the verification modes' own limits stand: TP 1, the row limit, no penalties at q_len > 1
    with pytest.raises(ValueError, match="tp_size 1"):
        DecodeStep(TINY, 4, 40, None, q_len=4, sampling=samp, tp_size=2, draft_probs=True)
    with pytest.raises(ValueError, match="max_rows"):
        DecodeStep(TINY, 40, 40, None, q_len=4, sampling=samp, draft_probs=True)
    with pytest.raises(ValueError, match="no penalties"):
        DecodeStep(TINY, 4, 40, None, q_len=4, sampling=SamplingParams(repetition=1.2), draft_probs=True)
