"""CPU tests of the finished-hypothesis set of beam search: the float64 reference (tests/beam_hyps_oracle.py) on hand-worked
cases, the argument checks of b200_beam_hypotheses_update / _finalize (rejected on the host before any CUDA call), and the
arguments DecodeStep's beam mode rejects with an eos_id."""
import ctypes

import numpy as np
import pytest

from rtp_llm_b200 import _lib
from tests.beam_hyps_oracle import FALSE, NEVER, TRUE, Hyps, hyp_score, parse_state

NINF = -np.inf
EOS = 9


def _full(W, scores, alpha=0.0, max_len=8):
    """A set holding one hypothesis of a single token per score (L 1, so score = cum at any alpha)."""
    h = Hyps(W, max_len)
    for s in scores:
        assert h.add(s, [EOS], alpha)
    return h


# ---------------------------------------------------------------------------------------------------- the reference
def test_fill_then_replace_the_worst():
    h = _full(3, [-2.0, -1.0, -3.0])
    assert [x["score"] for x in h.slots] == [-2.0, -1.0, -3.0] and h.next_order == 3
    assert h.add(-1.5, [4, EOS], 0.0)                         # beats the worst (-3.0, slot 2): takes its slot
    assert [x["score"] for x in h.slots] == [-2.0, -1.0, -1.5]
    assert h.slots[2]["order"] == 3 and h.slots[2]["tokens"] == [4, EOS] and h.slots[2]["len"] == 2
    assert not h.add(-5.0, [EOS], 0.0)                        # below the worst: does not enter
    assert h.next_order == 4


def test_an_equal_score_does_not_enter():
    h = _full(2, [-1.0, -2.0])
    assert not h.add(-4.0, [3, EOS], 1.0)                     # cum -4 over L 2 at alpha 1 = -2.0: equal to the worst
    assert [x["score"] for x in h.slots] == [-1.0, -2.0] and h.next_order == 2


def test_eviction_among_equal_lowest_takes_the_earliest_inserted():
    h = _full(3, [-2.0, -1.0, -2.0])
    assert h.add(-1.5, [EOS], 0.0)
    assert [x["order"] for x in h.slots] == [3, 1, 2]         # slot 0 (order 0) went, slot 2 (order 2) stays
    assert h.add(-1.8, [EOS], 0.0)
    assert [x["order"] for x in h.slots] == [3, 1, 4]


@pytest.mark.parametrize("alpha, exp", [(0.0, -6.0), (1.0, -2.0), (2.0, -6.0 / 9.0), (-1.0, -18.0)])
def test_length_penalty(alpha, exp):
    assert hyp_score(-6.0, 3, alpha) == exp
    h = Hyps(2, 8)
    h.add(-6.0, [1, 2, EOS], alpha)
    assert h.slots[0]["score"] == exp and h.slots[0]["cum"] == -6.0 and h.slots[0]["len"] == 3


def _cands(W, tokens, parents, scores):
    pad = 2 * W - len(tokens)
    return (np.array(tokens + [0] * pad), np.array(parents + [0] * pad), np.array(scores + [NINF] * pad, np.float64))


def test_update_takes_eos_below_rank_w_only_with_a_finite_score():
    W = 2
    h = Hyps(W, 8)
    paths = [[5, 6], [7, 8]]
    # rank 0 EOS from beam 1, rank 1 not EOS, rank 2 EOS (>= W: ignored)
    h.update(*_cands(W, [EOS, 3, EOS, 4], [1, 0, 0, 0], [-1.0, -1.2, -1.3, -1.4]), paths, EOS, 1.0, FALSE)
    assert len(h.slots) == 1
    assert h.slots[0]["tokens"] == [7, 8, EOS] and h.slots[0]["len"] == 3 and h.slots[0]["score"] == -1.0 / 3
    h.update(*_cands(W, [EOS, EOS, 1, 2], [0, 1, 0, 0], [NINF, NINF, NINF, NINF]), paths, EOS, 1.0, FALSE)
    assert len(h.slots) == 1                                  # -inf EOS candidates never enter
    assert not h.done


def test_paths_longer_than_max_len_are_truncated_but_scored_whole():
    h = Hyps(1, 2)
    h.add(-3.0, [1, 2, EOS], 1.0)
    assert h.slots[0]["tokens"] == [1, 2] and h.slots[0]["len"] == 3 and h.slots[0]["score"] == -1.0


def test_early_stopping_true_is_done_when_full():
    W = 2
    h = Hyps(W, 8)
    paths = [[1], [2]]
    h.update(*_cands(W, [EOS, 3, 4, 5], [0, 0, 0, 0], [-1.0, -1.1, -1.2, -1.3]), paths, EOS, 1.0, TRUE)
    assert not h.done                                         # one of two
    h.update(*_cands(W, [3, EOS, 4, 5], [0, 1, 0, 0], [-0.1, -9.0, -9.1, -9.2]), paths, EOS, 1.0, TRUE)
    assert h.done


@pytest.mark.parametrize("alpha", [0.0, 1.0, 2.0, -1.0])
def test_early_stopping_false_compares_the_worst_with_the_best_attainable(alpha):
    W, paths = 2, [[1, 2], [3, 4]]                            # L of this step's candidates = 3
    h = _full(W, [-1.0, -2.0], alpha)
    best_done = -2.05 * 3.0 ** alpha                          # best / 3^alpha = -2.05 <= worst -2.0: done
    g = copy_of(h)
    g.update(*_cands(W, [3, 4, 5, 6], [0, 0, 0, 0], [best_done, -10, -11, -12]), paths, EOS, alpha, FALSE)
    assert g.done
    best_not = -1.9 * 3.0 ** alpha                            # best / 3^alpha = -1.9 > worst: a live beam could still win
    g = copy_of(h)
    g.update(*_cands(W, [3, 4, 5, 6], [0, 0, 0, 0], [best_not, -10, -11, -12]), paths, EOS, alpha, FALSE)
    assert not g.done


def copy_of(h):
    import copy
    return copy.deepcopy(h)


def test_early_stopping_never_uses_max_len_for_a_positive_penalty():
    W, paths, max_len = 2, [[1, 2], [3, 4]], 8
    h = _full(W, [-1.0, -2.0], 1.0, max_len)
    best = -12.0                                              # / L 3 = -4 (< worst -2: done under False); / max_len 8 = -1.5
    g = copy_of(h)
    g.update(*_cands(W, [3, 4, 5, 6], [0] * 4, [best, -20, -21, -22]), paths, EOS, 1.0, FALSE)
    assert g.done
    g = copy_of(h)
    g.update(*_cands(W, [3, 4, 5, 6], [0] * 4, [best, -20, -21, -22]), paths, EOS, 1.0, NEVER)
    assert not g.done                                         # -2 < -12 / 8
    g.update(*_cands(W, [3, 4, 5, 6], [0] * 4, [-16.0, -20, -21, -22]), paths, EOS, 1.0, NEVER)
    assert g.done                                             # -2 >= -16 / 8


@pytest.mark.parametrize("alpha", [0.0, -1.0])
def test_early_stopping_never_at_a_non_positive_penalty_is_the_false_test(alpha):
    W, paths = 2, [[1, 2], [3, 4]]
    h = _full(W, [-1.0, -2.0], alpha)
    for best in (-2.05 * 3.0 ** alpha, -1.9 * 3.0 ** alpha):
        a, b = copy_of(h), copy_of(h)
        c = _cands(W, [3, 4, 5, 6], [0] * 4, [best, -20, -21, -22])
        a.update(*c, paths, EOS, alpha, FALSE)
        b.update(*c, paths, EOS, alpha, NEVER)
        assert a.done == b.done == (best < -2.0 * 3.0 ** alpha)


def test_a_done_request_is_frozen():
    W = 2
    h = _full(W, [-1.0, -2.0])
    h.update(*_cands(W, [3, 4, 5, 6], [0] * 4, [-5.0, -6, -7, -8]), [[1], [2]], EOS, 0.0, FALSE)
    assert h.done
    before = copy_of(h.slots)
    h.update(*_cands(W, [EOS, EOS, 5, 6], [0, 1, 0, 0], [-0.1, -0.2, -7, -8]), [[1], [2]], EOS, 0.0, FALSE)
    assert h.slots == before and h.next_order == 2


def test_finalize_merges_live_beams_into_a_set_that_is_not_full():
    W = 3
    h = Hyps(W, 6)
    h.add(-3.0, [1, 2, EOS], 1.0)                             # score -1.0
    beam_cum = np.array([-1.5, -4.0, NINF])
    paths = [[4, 5, 6], [7, 8], [9]]                          # scores -0.5, -2.0; beam 2 dead
    out = h.finalize(3, beam_cum, paths, 1.0)
    np.testing.assert_array_equal(out["len"], [3, 3, 2])
    np.testing.assert_array_equal(out["score"], [-0.5, -1.0, -2.0])
    np.testing.assert_array_equal(out["cum"], [-1.5, -3.0, -4.0])
    np.testing.assert_array_equal(out["tokens"], [[4, 5, 6, -1, -1, -1], [1, 2, EOS, -1, -1, -1], [7, 8, -1, -1, -1, -1]])
    assert len(h.slots) == 1 and h.next_order == 1            # the set itself is unchanged
    out = h.finalize(2, beam_cum, paths, 1.0)
    np.testing.assert_array_equal(out["score"], [-0.5, -1.0])
    h.done = True                                             # done: the live beams are not merged
    out = h.finalize(2, beam_cum, paths, 1.0)
    np.testing.assert_array_equal(out["len"], [3, -1])
    assert out["score"][1] == NINF and out["cum"][1] == NINF and (out["tokens"][1] == -1).all()


def test_finalize_orders_equal_scores_by_insertion():
    h = _full(3, [-1.0, -2.0, -1.0])
    out = h.finalize(3, np.full(3, NINF), [[], [], []], 0.0)
    np.testing.assert_array_equal(out["cum"], [-1.0, -1.0, -2.0])
    assert h.slots[0]["order"] == 0 and h.slots[2]["order"] == 2


def test_parse_state_reads_the_documented_layout():
    W, max_len = 2, 3
    raw = np.zeros(2 * (16 + 16 * W + 4 * W * max_len), np.uint8)
    s = raw[: 16 + 16 * W + 4 * W * max_len]
    s[:16].view(np.int32)[:2] = [1, 5]
    m = s[16:16 + 16 * W]
    m.view(np.float32)[:2] = [-3.0, -1.5]
    m.view(np.int32)[2:4] = [2, 4]
    s[16 + 16 * W:].view(np.int32)[:2] = [7, EOS]
    got = parse_state(raw, 2, W, max_len)
    assert got[0] == dict(count=1, next_order=5, slots=[dict(cum=-3.0, score=-1.5, len=2, order=4, tokens=[7, EOS])])
    assert got[1] == dict(count=0, next_order=0, slots=[])


# ---------------------------------------------------------------------------------------------------- the C ABI
@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def p():
    buf = (ctypes.c_uint8 * (1 << 16))()
    p.keep = buf
    return ctypes.cast(buf, ctypes.c_void_p)


def _update(lib, p, B=2, W=4, eos=3, max_len=8, state_bytes=None, stride=16, gen_start=1, **null):
    a = dict(ct=p, cp=p, cs=p, hist=p, hl=p, lp=p, es=p, state=p, done=p)
    a.update(null)
    if state_bytes is None:
        state_bytes = lib.b200_beam_hypotheses_state_bytes(B, 4, 8)
    return lib.b200_beam_hypotheses_update(a["ct"], a["cp"], a["cs"], a["hist"], a["hl"], stride, gen_start, B, W, eos, a["lp"],
                                           a["es"], max_len, a["state"], state_bytes, a["done"], None)


def _finalize(lib, p, B=2, W=4, n=2, max_len=8, state_bytes=None, stride=16, gen_start=1, **null):
    a = dict(state=p, done=p, cum=p, hist=p, hl=p, lp=p, tok=p, len_=p, score=p, ocum=p)
    a.update(null)
    if state_bytes is None:
        state_bytes = lib.b200_beam_hypotheses_state_bytes(B, 4, 8)
    return lib.b200_beam_hypotheses_finalize(a["state"], state_bytes, a["done"], a["cum"], a["hist"], a["hl"], stride, gen_start,
                                             B, W, n, max_len, a["lp"], a["tok"], a["len_"], a["score"], a["ocum"], None)


def test_state_bytes_follow_the_documented_layout(lib):
    assert lib.b200_beam_hypotheses_state_bytes(3, 4, 8) == 3 * (16 + 16 * 4 + 4 * 4 * 8)
    assert lib.b200_beam_hypotheses_state_bytes(0, 4, 8) == 0
    for B, W, L in ((2, 0, 8), (2, 33, 8), (2, 4, 0), (-1, 4, 8)):
        assert lib.b200_beam_hypotheses_state_bytes(B, W, L) == 0


def test_update_argument_checks(lib, p):
    for name in ("ct", "cp", "cs", "hist", "hl", "lp", "es", "state", "done"):
        assert _update(lib, p, **{name: None}) == -1 and b"null" in lib.b200_last_error(), name
    for W in (0, 33):
        assert _update(lib, p, W=W) == -1 and b"beam_width" in lib.b200_last_error()
    assert _update(lib, p, max_len=0) == -1 and b"max_len" in lib.b200_last_error()
    assert _update(lib, p, eos=-1) == -1 and b"eos_id" in lib.b200_last_error()
    assert _update(lib, p, state_bytes=100) == -1 and b"state too small" in lib.b200_last_error()
    assert _update(lib, p, max_len=9) == -1 and b"state too small" in lib.b200_last_error()   # the state was sized for 8
    assert _update(lib, p, stride=0) == -1 and b"hist_stride" in lib.b200_last_error()
    assert _update(lib, p, gen_start=-1) == -1 and b"gen_start" in lib.b200_last_error()
    assert _update(lib, p, B=0, ct=None, state=None) == 0                                   # empty batch: no work


def test_finalize_argument_checks(lib, p):
    for name in ("state", "done", "cum", "hist", "hl", "lp", "tok", "len_", "score", "ocum"):
        assert _finalize(lib, p, **{name: None}) == -1 and b"null" in lib.b200_last_error(), name
    for W in (0, 33):
        assert _finalize(lib, p, W=W, n=1) == -1 and b"beam_width" in lib.b200_last_error()
    for n in (0, 5, -1):
        assert _finalize(lib, p, n=n) == -1 and b"n " in lib.b200_last_error()
    assert _finalize(lib, p, max_len=0) == -1 and b"max_len" in lib.b200_last_error()
    assert _finalize(lib, p, state_bytes=16) == -1 and b"state too small" in lib.b200_last_error()
    assert _finalize(lib, p, B=0, state=None) == 0


def test_ops_reject_bad_arguments_before_any_launch():
    import torch
    from rtp_llm_b200 import ops
    B, W, L = 2, 4, 8
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32)            # noqa: E731
    cand = dict(cand_token=i32(B, 2 * W), cand_parent=i32(B, 2 * W), cand_score=torch.zeros(B, 2 * W))
    args = dict(history=i32(B * W, 16), hist_len=i32(B * W), eos_id=3, length_penalty=torch.ones(B), early_stopping=i32(B),
                state=torch.zeros(int(_lib.load().b200_beam_hypotheses_state_bytes(B, W, L)), dtype=torch.uint8), done=i32(B),
                max_len=L)
    with pytest.raises(_lib.B200Error, match="state"):
        ops.beam_hypotheses_update(cand, **dict(args, max_len=L + 1))
    with pytest.raises(_lib.B200Error, match="history"):
        ops.beam_hypotheses_update(cand, **dict(args, history=i32(B, 16)))
    with pytest.raises(_lib.B200Error, match="length_penalty"):
        ops.beam_hypotheses_update(cand, **dict(args, length_penalty=torch.ones(B, dtype=torch.float64)))
    with pytest.raises(_lib.B200Error, match="early_stopping"):
        ops.beam_hypotheses_update(cand, **dict(args, early_stopping=i32(B + 1)))
    with pytest.raises(_lib.B200Error, match="eos_id"):
        ops.beam_hypotheses_update(cand, **dict(args, eos_id=-1))
    with pytest.raises(_lib.B200Error, match="cand_score"):
        ops.beam_hypotheses_update(dict(cand, cand_score=i32(B, 2 * W)), **args)
    fin = dict(state=args["state"], done=args["done"], beam_cum=torch.zeros(B, W), history=args["history"],
               hist_len=args["hist_len"], max_len=L, length_penalty=args["length_penalty"])
    for n in (0, W + 1):
        with pytest.raises(_lib.B200Error, match="n "):
            ops.beam_hypotheses_finalize(n=n, **fin)
    with pytest.raises(_lib.B200Error, match="done"):
        ops.beam_hypotheses_finalize(n=1, **dict(fin, done=i32(B + 1)))
    with pytest.raises(_lib.B200Error, match="unsupported"):
        ops.beam_hypotheses_state(2, 33, 8, "cpu")


def test_decode_step_rejects_bad_eos_arguments():
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    with pytest.raises(ValueError, match="eos_id"):
        DecodeStep(TINY, 4, 40, None, eos_id=5)                   # the greedy step has no hypotheses
    with pytest.raises(ValueError, match="eos_id"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, eos_id=TINY.vocab)
    with pytest.raises(ValueError, match="eos_id"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, eos_id=-1)
    with pytest.raises(ValueError, match="early_stopping"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, eos_id=5, early_stopping="sometimes")
    with pytest.raises(ValueError, match="length_penalty: 3 values for 4 requests"):
        DecodeStep(TINY, 4, 40, None, beam_width=2, eos_id=5, length_penalty=[1.0, 1.0, 1.0])


def test_beam_results_needs_an_eos_id():
    from rtp_llm_b200.decode_step import DecodeStep
    step = DecodeStep.__new__(DecodeStep)
    step.W, step.eos_id = 4, None
    with pytest.raises(ValueError, match="eos_id"):
        step.beam_results(2)
