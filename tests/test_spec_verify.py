"""CPU tests of speculative-token verification: the argument checks of the new entry points (rejected on the host before any
CUDA call), and the numpy reference spec_verify_np (tests/spec_oracle.py), whose chain rejection sampling must reproduce the
target distribution exactly (the property the reference's speculative-sampling kernel rests on)."""
import ctypes

import numpy as np
import pytest

from rtp_llm_b200 import _lib
from tests.spec_oracle import spec_verify_np


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def hostbuf():
    buf = (ctypes.c_uint8 * (1 << 16))()
    return buf, ctypes.cast(buf, ctypes.c_void_p)


def _attn_multi(lib, p, Hq, Hkv, q_len, D=128):
    return lib.b200_paged_decode_attn_multi(p, 0, p, Hq, Hkv, D, 2, q_len, 4, 256, 64, p, p, p, 1.0, p, 4096, None)


def test_attention_accepts_up_to_64_query_rows_and_names_the_limit(lib, hostbuf):
    _, p = hostbuf
    for Hq, Hkv, q_len in [(64, 1, 2), (13, 1, 5), (65, 1, 1)]:      # 128, 65, 65 rows
        assert _attn_multi(lib, p, Hq, Hkv, q_len) == -1
        assert b"64" in lib.b200_last_error(), lib.b200_last_error()
    assert lib.b200_paged_decode_attn(p, 0, p, 65, 1, 128, 2, 4, 256, 64, p, p, p, 1.0, p, 4096, None) == -1
    assert b"1..64" in lib.b200_last_error()
    assert _attn_multi(lib, p, 8, 1, 65) == -1 and b"q_len" in lib.b200_last_error()
    # the fused-rope entry still loads q into one 16-row tile
    assert lib.b200_paged_decode_attn_rope(p, 0, p, 17, 1, 128, 2, 4, 256, 64, p, p, p, 1.0, 10000.0, p, 4096, None) == -1
    assert b"1..16" in lib.b200_last_error()


def test_rope_append_multi_argument_checks(lib, hostbuf):
    _, p = hostbuf
    args = (0, 2, 4, 2, 128, 4, 16, 10000.0)
    assert lib.b200_rope_append_multi(None, p, p, p, p, *args, 2, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_rope_append_multi(p, p, p, p, p, *args, 0, None) == -1 and b"q_len" in lib.b200_last_error()


def test_spec_verify_argument_checks(lib, hostbuf):
    _, p = hostbuf
    assert lib.b200_spec_verify(None, p, None, p, None, 2, -1, 100, p, p, None) == -1 and b"num_draft" in lib.b200_last_error()
    assert lib.b200_spec_verify(None, p, None, p, None, 2, 3, 100, None, p, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_spec_verify(None, p, None, None, None, 2, 3, 100, p, p, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_spec_verify(None, None, None, p, None, 2, 3, 100, p, p, None) == -1 and b"target" in lib.b200_last_error()
    assert lib.b200_spec_verify(p, None, None, p, None, 2, 3, 100, p, p, None) == -1 and b"uniform" in lib.b200_last_error()
    assert lib.b200_spec_verify(None, p, p, p, None, 2, 3, 100, p, p, None) == -1 and b"draft_probs" in lib.b200_last_error()
    assert lib.b200_spec_verify(None, None, None, None, None, 0, 3, 100, None, None, None) == 0      # empty batch: no work


def test_decode_step_rejects_unsupported_verification_shapes():
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    with pytest.raises(ValueError, match="128"):
        DecodeStep(TINY, 33, 40, None, q_len=4)
    with pytest.raises(ValueError, match="tp_size"):
        DecodeStep(TINY, 4, 40, None, q_len=2, tp_size=2)
    with pytest.raises(ValueError, match="q_len"):
        DecodeStep(TINY, 4, 40, None, q_len=0)


# ---------------------------------------------------------------------------------------------------- the oracle
def _first_token(d, target, draft_probs, u0, u1):
    t = np.stack([target, target]).astype(np.float32)[None]                  # [1, n+1 = 2, V]: row 1 is never reached here
    dp = None if draft_probs is None else draft_probs.astype(np.float32)[None, None]
    out, _ = spec_verify_np(np.array([[d]]), target_probs=t, draft_probs=dp, uniform=np.array([[u0, u1]]))
    return int(out[0, 0])


def _accept_measure(d, target, draft_probs):
    """Measure of {u0 in [0, 1)} accepting draft d: the accept set is {u0 : fp32(u0) * p < q}, downward closed, so it is
    [0, b) with b the least float32 that rejects, found by bisection over the float32 bit patterns of [0, 1). After a
    rejection the residual has no mass at d (rejection needs q(d) < p(d)), so the first token is d iff d was accepted."""
    acc = lambda u: _first_token(d, target, draft_probs, u, 0.0) == d
    lo, hi = 0, int(np.float32(1.0).view(np.uint32))                      # invariant: lo accepts (or is 0), hi rejects
    if not acc(0.0):
        return 0.0
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if acc(float(np.uint32(mid).view(np.float32))):
            lo = mid
        else:
            hi = mid
    return float(np.uint32(hi).view(np.float32))


def _draw_measures(d, target, draft_probs):
    """Measure of {u1 in [0, 1)} giving each token after a rejection of d: the draw is monotone in u1, so each token owns an
    interval whose ends are found by bisection (float64) to 1e-15."""
    V = target.shape[0]
    u0 = 0.9999999                                                         # rejects whenever rejection is possible
    tok = lambda u: _first_token(d, target, draft_probs, u0, u)
    ends = []
    for x in range(V):
        lo, hi = 0.0, 1.0                                                  # least u with tok(u) > x
        if tok(0.0) > x:
            ends.append(0.0)
            continue
        while hi - lo > 1e-15:
            mid = 0.5 * (lo + hi)
            if tok(mid) > x:
                hi = mid
            else:
                lo = mid
        ends.append(hi)
    ends = np.array(ends)
    return np.diff(np.concatenate([[0.0], ends]))


CASES = [
    # draft distribution p (powers of two, so q / p is exact in float32), target q (dyadic)
    (np.array([0.5, 0.25, 0.125, 0.125]), np.array([5, 27, 12, 20]) / 64),
    (np.array([0.25, 0.25, 0.5, 0.0]), np.array([16, 0, 40, 8]) / 64),
    (np.array([0.5, 0.0, 0.25, 0.125, 0.0625, 0.0625, 0.0, 0.0]), np.array([3, 9, 1, 0, 30, 7, 4, 10]) / 64),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_reproduces_the_target_distribution_with_draft_probabilities(case):
    p, q = CASES[case]
    P = np.zeros(len(q))
    for d in range(len(p)):
        if p[d] == 0:
            continue
        a = _accept_measure(d, q, p)
        np.testing.assert_allclose(a, min(1.0, q[d] / p[d]), atol=1e-12)
        P[d] += p[d] * a
        if a < 1.0:
            P += p[d] * (1.0 - a) * _draw_measures(d, q, p)
    np.testing.assert_allclose(P, q, atol=1e-9, rtol=0)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_reproduces_the_target_distribution_with_deterministic_drafts(case):
    _, q = CASES[case]
    for d in range(len(q)):                       # whatever the (one-hot) draft is, the first token is distributed as q
        a = _accept_measure(d, q, None)
        np.testing.assert_allclose(a, q[d], atol=1e-12)
        P = np.zeros(len(q))
        P[d] += a
        if a < 1.0:
            P += (1.0 - a) * _draw_measures(d, q, None)
        np.testing.assert_allclose(P, q, atol=1e-9, rtol=0, err_msg=f"draft {d}")


def test_greedy_mode_equals_sampling_with_one_hot_targets():
    rng = np.random.default_rng(3)
    B, n, V = 64, 5, 50
    ids = rng.integers(0, V, (B, n + 1))
    drafts = np.where(rng.random((B, n)) < 0.7, ids[:, :n], rng.integers(0, V, (B, n)))
    onehot = np.zeros((B, n + 1, V), np.float32)
    np.put_along_axis(onehot, ids[..., None], 1.0, axis=-1)
    g = spec_verify_np(drafts, target_ids=ids)
    s = spec_verify_np(drafts, target_probs=onehot, uniform=rng.random((B, n + 1)).astype(np.float32))
    np.testing.assert_array_equal(g[0], s[0])
    np.testing.assert_array_equal(g[1], s[1])
    assert 0 < g[1].mean() < n


def test_drafts_with_the_target_probabilities_are_all_accepted():
    rng = np.random.default_rng(4)
    B, n, V = 32, 4, 40
    t = rng.random((B, n + 1, V)).astype(np.float32) ** 4
    t /= t.sum(-1, keepdims=True)
    t64 = t.astype(np.float64)
    drafts = np.array([[rng.choice(V, p=t64[b, i] / t64[b, i].sum()) for i in range(n)] for b in range(B)])
    out, acc = spec_verify_np(drafts, target_probs=t, draft_probs=t[:, :n].copy(),
                              uniform=(rng.random((B, n + 1)) * 0.999).astype(np.float32))
    assert (acc == n).all()
    np.testing.assert_array_equal(out[:, :n], drafts)
    assert (out[:, n] >= 0).all()
