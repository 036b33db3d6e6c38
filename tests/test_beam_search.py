"""CPU tests of beam search: the argument checks of b200_beam_search_step and b200_ban_repeat_ngram (rejected on the host
before any CUDA call), the shapes DecodeStep's beam mode rejects, and the float64 reference (tests/beam_oracle.py) on
hand-made cases."""
import ctypes

import numpy as np
import pytest

from rtp_llm_b200 import _lib
from tests.beam_oracle import banned_np, beam_scores_np, beam_step_np, next_from_candidates

NINF = -np.inf


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def p():
    buf = (ctypes.c_uint8 * (1 << 16))()
    p.keep = buf
    return ctypes.cast(buf, ctypes.c_void_p)


def _beam(lib, p, B=2, W=4, V=1000, dtype=0, ws_bytes=1 << 16, **null):
    a = dict(logits=p, cum=p, ct=p, cp=p, cs=p, nt=p, np_=p, nc=p, ws=p)
    a.update(null)
    return lib.b200_beam_search_step(a["logits"], dtype, a["cum"], B, W, V, -1, a["ct"], a["cp"], a["cs"], a["nt"], a["np_"], a["nc"],
                                     a["ws"], ws_bytes, None)


def test_beam_search_step_argument_checks(lib, p):
    for name in ("logits", "cum", "ct", "cp", "cs", "nt", "np_", "nc"):
        assert _beam(lib, p, **{name: None}) == -1 and b"null" in lib.b200_last_error(), name
    for W in (0, 33, -1):
        assert _beam(lib, p, W=W) == -1 and b"beam_width" in lib.b200_last_error()
    assert _beam(lib, p, W=4, V=7) == -1 and b">= 2 * beam_width" in lib.b200_last_error()
    assert _beam(lib, p, dtype=3) == -1 and b"dtype" in lib.b200_last_error()
    assert _beam(lib, p, W=32, V=262145) == -1 and b"row merge" in lib.b200_last_error()
    assert _beam(lib, p, ws_bytes=16) == -1 and b"workspace too small" in lib.b200_last_error()
    assert _beam(lib, p, ws=None) == -1 and b"workspace" in lib.b200_last_error()
    assert _beam(lib, p, B=0, logits=None) == 0                           # empty batch: no work
    assert lib.b200_beam_search_step_workspace_bytes(8, 4, 128256) > 0
    assert lib.b200_beam_search_step_workspace_bytes(8, 33, 128256) == 0
    assert lib.b200_beam_search_step_workspace_bytes(8, 4, 7) == 0


def test_ban_repeat_ngram_argument_checks(lib, p):
    assert lib.b200_ban_repeat_ngram(None, 0, 2, 100, p, p, 8, p, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 0, 2, 100, None, p, 8, p, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 0, 2, 100, p, None, 8, p, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 0, 2, 100, p, p, 8, None, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 5, 2, 100, p, p, 8, p, None) == -1 and b"dtype" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 0, 2, 0, p, p, 8, p, None) == -1 and b"vocab" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(p, 0, 2, 100, p, p, 0, p, None) == -1 and b"hist_stride" in lib.b200_last_error()
    assert lib.b200_ban_repeat_ngram(None, 0, 0, 100, None, None, 8, None, None) == 0    # no rows: no work


def test_ops_reject_bad_arguments_before_any_launch():
    import torch
    from rtp_llm_b200 import ops
    x = torch.zeros(8, 100)
    with pytest.raises(_lib.B200Error, match="beam_width"):
        ops.beam_search_step(x, torch.zeros(2, 4), 33)
    with pytest.raises(_lib.B200Error, match="B \\* 3"):
        ops.beam_search_step(x, torch.zeros(2, 4), 3)
    with pytest.raises(_lib.B200Error, match="2 \\* beam_width"):
        ops.beam_search_step(torch.zeros(8, 7), torch.zeros(2, 4), 4)
    with pytest.raises(_lib.B200Error, match="fp16, bf16 or fp32"):
        ops.beam_search_step(x.double(), torch.zeros(2, 4), 4)
    with pytest.raises(_lib.B200Error, match="cum_log_probs"):
        ops.beam_search_step(x, torch.zeros(2, 4, dtype=torch.float64), 4)
    h = torch.zeros(8, 4, dtype=torch.int32)
    n = torch.zeros(8, dtype=torch.int32)
    with pytest.raises(_lib.B200Error, match="fp16, bf16 or fp32"):
        ops.ban_repeat_ngram(x.long(), h, n, n)
    with pytest.raises(_lib.B200Error, match="history"):
        ops.ban_repeat_ngram(x, h.long(), n, n)
    with pytest.raises(_lib.B200Error, match="ngram_size"):
        ops.ban_repeat_ngram(x, h, n, n[:3])


def test_decode_step_rejects_unsupported_beam_shapes():
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    with pytest.raises(ValueError, match="128"):
        DecodeStep(TINY, 33, 40, None, beam_width=4)
    with pytest.raises(ValueError, match="tp_size"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, tp_size=2)
    with pytest.raises(ValueError, match="q_len"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, q_len=2)
    with pytest.raises(ValueError, match="beam_width"):
        DecodeStep(TINY, 4, 40, None, beam_width=33)
    with pytest.raises(ValueError, match="no_repeat_ngram"):      # the greedy step has no ban: not silently ignored
        DecodeStep(TINY, 4, 40, None, no_repeat_ngram=3)
    with pytest.raises(ValueError, match="max_new_tokens"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, max_new_tokens=40)


def test_beam_steps_past_max_new_tokens_are_refused():
    """The page-table rows end max_new_tokens steps after the prompt: one more step raises before it launches anything."""
    from rtp_llm_b200.decode_step import DecodeStep
    step = DecodeStep.__new__(DecodeStep)
    step.W, step.max_new_tokens, step.beam_steps = 4, 2, 0
    step._count_beam_step()
    step._count_beam_step()
    with pytest.raises(ValueError, match="max_new_tokens 2"):
        step._count_beam_step()
    with pytest.raises(ValueError, match="max_new_tokens 2"):
        step.replay()                                              # the graph path counts too, before it replays
    step.W, step.beam_steps = 1, 5                                 # the greedy step is never limited
    step._count_beam_step()


def test_decode_step_beam_mode_is_not_a_program():
    """build_program() refuses a beam step before it records anything (the fork is torch index ops)."""
    from rtp_llm_b200.decode_step import DecodeStep
    step = DecodeStep.__new__(DecodeStep)
    step.tp_size, step.q_len, step.W = 1, 1, 4
    with pytest.raises(ValueError, match="program"):
        step.build_program()


# ---------------------------------------------------------------------------------------------------- the oracle
def test_oracle_breaks_ties_by_flat_index():
    # two beams, equal cum, identical rows: every score appears twice; the lower flat index (beam 0) ranks first
    row = np.array([0.0, 3.0, 1.0, 3.0, 2.0, -1.0])
    r = beam_step_np(np.stack([row, row]), np.zeros((1, 2)))
    np.testing.assert_array_equal(r["cand_token"][0], [1, 3, 1, 3])
    np.testing.assert_array_equal(r["cand_parent"][0], [0, 0, 1, 1])
    np.testing.assert_array_equal(r["next_token"][0], [1, 3])
    np.testing.assert_array_equal(r["next_parent"][0], [0, 0])
    lse = np.log(np.exp(row).sum())
    np.testing.assert_allclose(r["cand_score"][0], 3.0 - lse)


def test_oracle_skips_eos_inside_the_top_w():
    rows = np.array([[6.0, 4.0, 0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 3.0, 0.0, 1.0]])
    r = beam_step_np(rows, np.zeros((1, 2)), eos_id=0)
    s = beam_scores_np(rows, np.zeros((1, 2)))[0]
    ranked = sorted(((-s[i, v], i * 6 + v) for i in range(2) for v in range(6)))
    flat = [f for _, f in ranked[:4]]
    np.testing.assert_array_equal(r["cand_token"][0], [f % 6 for f in flat])
    assert r["cand_token"][0, 0] == 0                                   # EOS ranks first: a finished hypothesis
    assert 0 not in r["next_token"][0]
    nt, npar, nc = next_from_candidates(r["cand_token"], r["cand_parent"], r["cand_score"], 2, eos_id=0)
    np.testing.assert_array_equal(nt, r["next_token"])
    np.testing.assert_array_equal(npar, r["next_parent"])
    np.testing.assert_array_equal(nc, r["next_cum"])


def test_oracle_first_step_only_beam_zero_contributes():
    rng = np.random.default_rng(0)
    W, V = 4, 50
    rows = rng.standard_normal((W, V))
    cum = np.array([[0.0, NINF, NINF, NINF]])
    r = beam_step_np(rows, cum)
    assert (r["cand_parent"][0] == 0).all()
    np.testing.assert_array_equal(r["cand_token"][0], np.argsort(-rows[0], kind="stable")[:2 * W])
    # with fewer than 2W finite candidates the -inf ones fill up by flat index: beam 0's lowest masked ids first
    rows[0, 3:] = NINF
    r = beam_step_np(rows, cum)
    assert np.isfinite(r["cand_score"][0, :3]).all() and np.isneginf(r["cand_score"][0, 3:]).all()
    np.testing.assert_array_equal(r["cand_token"][0, 3:], [3, 4, 5, 6, 7])
    assert (r["cand_parent"][0] == 0).all()


def test_oracle_masked_logits_rank_last_by_index():
    rows = np.full((2, 4), NINF)
    rows[1, 2] = 0.0
    r = beam_step_np(rows, np.zeros((1, 2)))
    np.testing.assert_array_equal(r["cand_token"][0], [2, 0, 1, 2])
    np.testing.assert_array_equal(r["cand_parent"][0], [1, 0, 0, 0])
    assert r["cand_score"][0, 0] == 0.0 and np.isneginf(r["cand_score"][0, 1:]).all()


def test_ngram_oracle_edge_cases():
    V = 10
    h = np.array([[1, 2, 3, 1, 2, 0, 0, 0],     # n 3, suffix (1, 2): bans 3
                  [5, 5, 5, 5, 0, 0, 0, 0],     # n 2, overlapping matches of (5): bans 5
                  [7, 1, 9, 0, 0, 0, 0, 0],     # n 1: every token of the history
                  [4, 4, 0, 0, 0, 0, 0, 0],     # L = 2 < n = 3: nothing
                  [-3, 12, 1, -3, 12, 0, 0, 0],  # n 3, suffix (-3, 12) matches at 0: bans 1; out-of-range ids never banned
                  [12, 2, 12, 0, 0, 0, 0, 0],   # n 2: suffix (12) matches at 0, bans 2; the out-of-range 12 itself is not
                  [1, 2, 3, 1, 2, 0, 0, 0]])    # n 0: off
    L = np.array([5, 4, 3, 2, 5, 3, 5])
    n = np.array([3, 2, 1, 3, 3, 2, 0])
    got = banned_np(h, L, n, V)
    exp = [[3], [5], [1, 7, 9], [], [1], [2], []]
    for r in range(len(exp)):
        np.testing.assert_array_equal(got[r], exp[r], err_msg=f"row {r}")
    # an n-gram that is the whole history has no earlier start: nothing to ban
    assert banned_np(np.array([[1, 2, 3]]), [3], [3], V)[0].size == 0
    # hist_len beyond the stride is clamped to it
    np.testing.assert_array_equal(banned_np(np.array([[6, 6]]), [9], [2], V)[0], [6])
