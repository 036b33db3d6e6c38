"""CPU tests of sampled decoding: the argument checks of b200_token_logprobs and ops.token_logprobs (rejected on the host before
any CUDA call), the float64 log-prob reference (tests/logprob_oracle.py) on hand-made cases, the step's uniforms, and the
DecodeStep shapes the sampling mode rejects."""
import ctypes

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams, sampling_uniforms
from tests.logprob_oracle import log_softmax_np, token_logprobs_np

NINF = -np.inf


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def p():
    buf = (ctypes.c_uint8 * (1 << 16))()
    p.keep = buf
    return ctypes.cast(buf, ctypes.c_void_p)


def _lp(lib, p, rows=4, V=1000, top_n=5, dtype=0, ws_bytes=1 << 16, **null):
    a = dict(logits=p, tokens=p, tlp=p, ids=p, lps=p, ws=p)
    a.update(null)
    return lib.b200_token_logprobs(a["logits"], dtype, rows, V, top_n, a["tokens"], a["tlp"], a["ids"], a["lps"], a["ws"], ws_bytes,
                                   None)


def test_token_logprobs_argument_checks(lib, p):
    for name in ("logits", "tlp", "ids", "lps"):
        assert _lp(lib, p, **{name: None}) == -1 and b"null" in lib.b200_last_error(), name
    for n in (-1, 65):
        assert _lp(lib, p, top_n=n) == -1 and b"top_n" in lib.b200_last_error()
    assert _lp(lib, p, V=4, top_n=5) == -1 and b"top_n" in lib.b200_last_error()               # more than the vocabulary
    assert _lp(lib, p, V=300000, top_n=64) == -1 and b"row merge" in lib.b200_last_error()
    assert _lp(lib, p, dtype=3) == -1 and b"dtype" in lib.b200_last_error()
    assert _lp(lib, p, V=0) == -1 and b"vocab" in lib.b200_last_error()
    assert _lp(lib, p, rows=65536) == -1 and b"rows" in lib.b200_last_error()
    assert _lp(lib, p, ws_bytes=16) == -1 and b"workspace too small" in lib.b200_last_error()
    assert _lp(lib, p, ws=None) == -1 and b"workspace" in lib.b200_last_error()
    assert _lp(lib, p, rows=0, logits=None) == 0                                            # no rows: no work
    assert lib.b200_token_logprobs_workspace_bytes(32, 128256, 20) > 0
    assert lib.b200_token_logprobs_workspace_bytes(32, 128256, 0) > 0
    assert lib.b200_token_logprobs_workspace_bytes(32, 128256, 65) == 0
    assert lib.b200_token_logprobs_workspace_bytes(32, 10, 11) == 0
    # top_n 0 needs no top outputs; the workspace grows with top_n
    assert lib.b200_token_logprobs_workspace_bytes(32, 128256, 20) > lib.b200_token_logprobs_workspace_bytes(32, 128256, 5)


def test_ops_token_logprobs_rejects_bad_arguments_before_any_launch():
    x = torch.zeros(8, 100)
    with pytest.raises(_lib.B200Error, match="fp16, bf16 or fp32"):
        ops.token_logprobs(x.double(), 5)
    with pytest.raises(_lib.B200Error, match="fp16, bf16 or fp32"):
        ops.token_logprobs(x.long(), 5)
    with pytest.raises(_lib.B200Error, match=r"\[rows, V\]"):
        ops.token_logprobs(torch.zeros(8), 5)
    for n in (-1, 65):
        with pytest.raises(_lib.B200Error, match="top_n"):
            ops.token_logprobs(x, n)
    with pytest.raises(_lib.B200Error, match="top_n"):
        ops.token_logprobs(torch.zeros(2, 10), 11)
    with pytest.raises(_lib.B200Error, match="top_n"):
        ops.token_logprobs(torch.zeros(2, 300000, dtype=torch.float16), 64)
    with pytest.raises(_lib.B200Error, match="tokens"):
        ops.token_logprobs(x, 5, tokens=torch.zeros(8, dtype=torch.int64))
    with pytest.raises(_lib.B200Error, match="tokens"):
        ops.token_logprobs(x, 5, tokens=torch.zeros(7, dtype=torch.int32))
    with pytest.raises(_lib.B200Error, match="top_ids"):
        ops.token_logprobs(x, 5, out=dict(top_ids=torch.zeros(8, 4, dtype=torch.int32)))
    with pytest.raises(_lib.B200Error, match="top_logprobs"):
        ops.token_logprobs(x, 5, out=dict(top_logprobs=torch.zeros(8, 5, dtype=torch.float16)))
    with pytest.raises(_lib.B200Error, match="workspace"):
        ops.token_logprobs(x, 5, workspace=torch.zeros(16, dtype=torch.uint8))
    with pytest.raises(_lib.B200Error, match="unsupported shape"):
        ops.token_logprobs_workspace(8, 100, 65, "cpu")


def test_ops_sample_checks_preallocated_outputs():
    x = torch.zeros(4, 10)
    k, tp, u = torch.zeros(4, dtype=torch.int32), torch.ones(4), torch.zeros(4)
    with pytest.raises(_lib.B200Error, match="token"):
        ops.sample(x, k, tp, u, out=dict(token=torch.zeros(4, dtype=torch.int64)))
    with pytest.raises(_lib.B200Error, match="probs"):
        ops.sample(x, k, tp, u, out=dict(probs=torch.zeros(4, 9)))


# ---------------------------------------------------------------------------------------------------- the oracle
def test_oracle_log_softmax_and_ties():
    row = np.array([0.0, 3.0, 1.0, 3.0, 2.0, NINF])
    r = token_logprobs_np(row[None], 4, tokens=[4])
    lse = np.log(np.exp(row[:5]).sum())
    np.testing.assert_allclose(r["lp"][0], row - lse)
    np.testing.assert_array_equal(r["top_ids"][0], [1, 3, 4, 2])            # the tie 1 / 3 goes to the lower id first
    np.testing.assert_allclose(r["top_logprobs"][0], row[[1, 3, 4, 2]] - lse)
    np.testing.assert_allclose(r["token_logprob"], [2.0 - lse])
    np.testing.assert_allclose(np.exp(r["lp"]).sum(), 1.0)


def test_oracle_edge_rows():
    x = np.array([[5.0] * 6,                                   # all equal: every lp is -log V, ids in order
                  [np.nan, 1.0, NINF, 1.0, NINF, 0.0],         # NaN counts as -inf
                  [NINF] * 6])                                 # no finite logit: NaN
    r = token_logprobs_np(x, 3, tokens=[2, 0, 1])
    np.testing.assert_allclose(r["top_logprobs"][0], [-np.log(6)] * 3)
    np.testing.assert_array_equal(r["top_ids"][0], [0, 1, 2])
    np.testing.assert_array_equal(r["top_ids"][1], [1, 3, 5])
    assert np.isneginf(r["token_logprob"][1]) and np.isnan(r["token_logprob"][2])
    assert np.isnan(log_softmax_np(x[2:])).all()
    assert np.isnan(token_logprobs_np(x[:1], 0, tokens=[6])["token_logprob"][0])     # an id outside the vocabulary
    assert token_logprobs_np(x, 0)["top_ids"].shape == (3, 0)


# ---------------------------------------------------------------------------------------------------- the step
def test_uniforms_follow_from_seed_and_step():
    a = sampling_uniforms(3, 0, 64)
    assert a.dtype == torch.float32 and torch.equal(a, sampling_uniforms(3, 0, 64))
    assert torch.equal(sampling_uniforms(3, 0, 8), a[:8])                  # row i does not depend on the row count
    assert not torch.equal(a, sampling_uniforms(3, 1, 64)) and not torch.equal(a, sampling_uniforms(4, 0, 64))
    u = torch.cat([sampling_uniforms(7, t, 128) for t in range(64)])
    assert float(u.min()) >= 0.0 and float(u.max()) < 1.0
    assert abs(float(u.mean()) - 0.5) < 0.02 and u.unique().numel() > 0.99 * u.numel()


def test_decode_step_rejects_unsupported_sampling_shapes():
    sp = SamplingParams(top_k=50, top_p=0.9)
    with pytest.raises(ValueError, match="tp_size"):
        DecodeStep(TINY, 4, 40, None, sampling=sp, tp_size=2)
    with pytest.raises(ValueError, match="beam_width"):
        DecodeStep(TINY, 4, 40, None, sampling=sp, beam_width=2)
    with pytest.raises(ValueError, match="128"):
        DecodeStep(TINY, 129, 40, None, sampling=sp)
    with pytest.raises(ValueError, match="128"):
        DecodeStep(TINY, 33, 40, None, sampling=sp, q_len=4)
    for bad in (dict(sampling=SamplingParams(repetition=1.2)), dict(sampling=SamplingParams(presence=[0.0, 0.5, 0.0, 0.0])),
                dict(sampling=SamplingParams(frequency=0.1)), dict(sampling=sp, no_repeat_ngram=2)):
        with pytest.raises(ValueError, match="drafts 0..j-1"):
            DecodeStep(TINY, 4, 40, None, q_len=2, **bad)
    with pytest.raises(ValueError, match="max_new_tokens"):
        DecodeStep(TINY, 4, 40, None, sampling=sp, max_new_tokens=40)
    with pytest.raises(ValueError, match="logprobs"):
        DecodeStep(TINY, 4, 40, None, sampling=sp, logprobs=65)
    with pytest.raises(ValueError, match="logprobs"):
        DecodeStep(TINY, 4, 40, None, logprobs=5)                      # log-probs come with the sampling mode
    assert SamplingParams(repetition=[1.0, 1.0]).has_penalties() is False
    assert SamplingParams(repetition=[1.0, 1.1]).has_penalties() and SamplingParams(frequency=0.2).has_penalties()


def test_ban_without_beam_or_sampling_still_raises():
    with pytest.raises(ValueError, match="no_repeat_ngram 3 needs beam search"):
        DecodeStep(TINY, 4, 40, None, no_repeat_ngram=3)


def test_sampled_steps_past_max_new_tokens_are_refused():
    step = DecodeStep.__new__(DecodeStep)
    step.W, step.sample_advances, step.max_new_tokens, step.beam_steps = 1, True, 2, 0
    step._count_beam_step()
    step._count_beam_step()
    with pytest.raises(ValueError, match="max_new_tokens 2"):
        step._count_beam_step()
    with pytest.raises(ValueError, match="max_new_tokens 2"):
        step.replay()


def test_sampling_step_is_not_a_program():
    step = DecodeStep.__new__(DecodeStep)
    step.tp_size, step.q_len, step.W, step.samp = 1, 1, 1, SamplingParams()
    with pytest.raises(ValueError, match="program"):
        step.build_program()
