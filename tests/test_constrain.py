"""CPU tests of constrained decoding: the argument checks of b200_constrain_logits and of b200_sample's min_p position (rejected
on the host before any CUDA call), the ops host checks and the logit-bias CSR builder, the numpy contract
(tests/constrain_oracle.py) on hand-made cases, and what DecodeStep rejects or validates in set_constraints()."""
import ctypes

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams
from tests.constrain_oracle import NEG_INF, allowed, constrain, min_p_kept, round_to, to_f32


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def p():
    buf = (ctypes.c_uint8 * (1 << 16))()
    p.keep = buf
    return ctypes.cast(buf, ctypes.c_void_p)


def _cl(lib, p, rows=4, V=1000, dtype=0, stride=32, **kw):
    a = dict(logits=p, mask=p, off=p, ids=p, vals=p)
    a.update(kw)
    return lib.b200_constrain_logits(a["logits"], dtype, rows, V, a["mask"], stride, a["off"], a["ids"], a["vals"], None)


def test_constrain_logits_argument_checks(lib, p):
    assert _cl(lib, p, logits=None) == -1 and b"null" in lib.b200_last_error()
    assert _cl(lib, p, ids=None) == -1 and b"null" in lib.b200_last_error()
    assert _cl(lib, p, vals=None) == -1 and b"null" in lib.b200_last_error()
    assert _cl(lib, p, mask=None, off=None) == -1 and b"neither" in lib.b200_last_error()
    assert _cl(lib, p, dtype=3) == -1 and b"dtype" in lib.b200_last_error()
    assert _cl(lib, p, dtype=-1) == -1 and b"dtype" in lib.b200_last_error()
    assert _cl(lib, p, V=0) == -1 and b"vocab" in lib.b200_last_error()
    for rows in (0, 65536):
        assert _cl(lib, p, rows=rows) == -1 and b"rows" in lib.b200_last_error()
    assert _cl(lib, p, V=1000, stride=31) == -1 and b"mask_stride" in lib.b200_last_error()     # ceil(1000 / 32) = 32
    assert _cl(lib, p, V=1025, stride=32) == -1 and b"mask_stride" in lib.b200_last_error()


def test_sample_takes_min_p_after_top_p(lib, p):
    """b200_sample(logits, rows, vocab, history, hist_len, hist_stride, count_ws, temperature, repetition, presence, frequency,
    top_k, top_p, min_p, uniform, process, token_out, token_prob_out, probs_out, stream): uniform sits after min_p."""
    args = [p, 4, 100, None, None, 0, None, None, None, None, None, p, p, p, p, None, p, None, None, None]
    assert len(args) == len(_lib.SIGNATURES["b200_sample"][1])
    bad = list(args)
    bad[14] = None                                   # uniform
    assert lib.b200_sample(*bad) == -1 and b"null" in lib.b200_last_error()
    bad = list(args)
    bad[12] = None                                   # top_p
    assert lib.b200_sample(*bad) == -1 and b"null" in lib.b200_last_error()


# ---------------------------------------------------------------------------------------------------- ops host checks
def test_ops_constrain_logits_rejects_bad_arguments_before_any_launch():
    x = torch.zeros(4, 100, dtype=torch.float16)
    m = torch.zeros(4, 4, dtype=torch.int32)
    bias = (torch.zeros(5, dtype=torch.int32), torch.zeros(3, dtype=torch.int32), torch.zeros(3))
    with pytest.raises(_lib.B200Error, match="fp16, bf16 or fp32"):
        ops.constrain_logits(x.double(), m)
    with pytest.raises(_lib.B200Error, match=r"\[rows, V\]"):
        ops.constrain_logits(torch.zeros(100, dtype=torch.float16), m)
    with pytest.raises(_lib.B200Error, match="rows"):
        ops.constrain_logits(torch.zeros(0, 100, dtype=torch.float16), m)
    with pytest.raises(_lib.B200Error, match="bitmask, a logit_bias"):
        ops.constrain_logits(x)
    for bad in (m[:, :3], m[:3], m.long(), m.view(-1)):
        with pytest.raises(_lib.B200Error, match="bitmask must be int32"):
            ops.constrain_logits(x, bad)
    for bad in ((bias[0][:4],) + bias[1:], (bias[0].long(),) + bias[1:], (bias[0], bias[1].long(), bias[2]),
                (bias[0], bias[1], bias[2].half()), (bias[0], bias[1], bias[2][:2])):
        with pytest.raises(_lib.B200Error, match="bias"):
            ops.constrain_logits(x, logit_bias=bad)
    with pytest.raises(_lib.B200Error, match="CUDA"):                       # shapes pass; host tensors do not
        ops.constrain_logits(x, m, bias)


def test_ops_sample_checks_min_p():
    x = torch.zeros(4, 10)
    k, tp, u = torch.zeros(4, dtype=torch.int32), torch.ones(4), torch.zeros(4)
    with pytest.raises(_lib.B200Error, match="min_p must be fp32"):
        ops.sample(x, k, tp, u, min_p=torch.zeros(3))
    with pytest.raises(_lib.B200Error, match="min_p must be fp32"):
        ops.sample(x, k, tp, u, min_p=torch.zeros(4, dtype=torch.float64))
    for bad in (-0.01, 1.01, float("nan")):
        with pytest.raises(_lib.B200Error, match=r"min_p must be in \[0, 1\]"):
            ops.sample(x, k, tp, u, min_p=torch.tensor([0.1, bad, 0.0, 1.0]))
    with pytest.raises(_lib.B200Error, match="CUDA"):                       # in range; host tensors do not pass
        ops.sample(x, k, tp, u, min_p=torch.tensor([0.0, 0.5, 1.0, 0.2]))


def test_logit_bias_csr():
    off, ids, vals = ops.logit_bias_csr([{5: 1.5, 0: -2}, {}, {99: float("-inf"), 7: 1e40}], 100)
    assert off.dtype == ids.dtype == torch.int32 and vals.dtype == torch.float32
    assert off.tolist() == [0, 2, 2, 4] and ids.tolist() == [5, 0, 99, 7]
    assert vals.tolist() == [1.5, -2.0, float("-inf"), float("inf")]            # 1e40 is +inf in fp32
    assert ops.logit_bias_csr([{np.int64(3): np.float32(0.25)}], 4)[1].tolist() == [3]       # numpy scalars are numbers
    off, ids, vals = ops.logit_bias_csr([], 10)
    assert off.tolist() == [0] and ids.numel() == 0 and vals.numel() == 0
    for bad in ({100: 1.0}, {-1: 1.0}, {True: 1.0}, {"5": 1.0}, {2.0: 1.0}):
        with pytest.raises(_lib.B200Error, match="token id"):
            ops.logit_bias_csr([{}, bad], 100)
    for bad in (float("nan"), "1.0", None, True, 1j):
        with pytest.raises(_lib.B200Error, match="not a number"):
            ops.logit_bias_csr([{3: bad}], 100)


# ---------------------------------------------------------------------------------------------------- the oracle
def _mask(rows, V, allowed_tokens):
    m = np.zeros((rows, (V + 31) // 32), np.uint32)
    for r, toks in enumerate(allowed_tokens):
        for t in toks:
            m[r, t >> 5] |= np.uint32(1) << np.uint32(t & 31)
    return m.view(np.int32)


def test_oracle_bit_order_is_lsb_first():
    m = np.array([[1, -2147483648, 0x10]], np.int32)                           # bit 0 of word 0, bit 31 of word 1, bit 4 of word 2
    a = allowed(m, 96)
    assert np.flatnonzero(a[0]).tolist() == [0, 63, 68]
    assert allowed(np.array([[-1]], np.int32), 32).all()                      # an all-ones word allows its 32 tokens


def test_oracle_partial_last_word_and_bits_past_vocab():
    V = 40                                                                    # word 1 holds tokens 32..39 and 24 bits past V
    m = np.array([[0, -1], [-1, 0], [0, 0x100]], np.int32)                    # row 2: bit 8 of word 1 = token 40, past V
    a = allowed(m, V)
    assert np.flatnonzero(a[0]).tolist() == list(range(32, 40))
    assert np.flatnonzero(a[1]).tolist() == list(range(32))
    assert not a[2].any()                                                     # a bit past V allows nothing
    x = round_to(np.arange(2 * V, dtype=np.float32).reshape(2, V), "fp16")
    y, _ = constrain(x, "fp16", m[:2])
    assert (y[0, :32] == NEG_INF["fp16"]).all() and (y[0, 32:] == x[0, 32:]).all()
    assert (y[1, 32:] == NEG_INF["fp16"]).all() and (y[1, :32] == x[1, :32]).all()
    wide = np.concatenate([m[:2], np.full((2, 3), 12345, np.int32)], axis=1)   # a larger stride: its extra words are not read
    assert np.array_equal(allowed(wide, V), a[:2])


@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp32"])
def test_oracle_bias_arithmetic(dtype):
    V = 8
    vals = np.array([1.0, 2.0, -3.0, np.nan, np.inf, -np.inf, 0.5, 100.0], np.float32)
    x = round_to(vals[None], dtype)
    m = _mask(1, V, [[0, 1, 2, 3, 4, 6, 7]])                                  # token 5 masked
    off, ids = np.array([0, 8]), np.array([5, 0, 1, 3, 4, 6, 7, 9])          # id 9 is outside the vocabulary
    b = np.array([7.0, 1e-4, -np.inf, 1.0, -np.inf, 0.1, 7e4, 1.0], np.float32)
    y, biased = constrain(x, dtype, m, off, ids, b)
    f = to_f32(y, dtype)[0]
    assert y[0, 5] == NEG_INF[dtype] and not biased[0, 5]                    # a bias on a masked token has no effect
    assert y[0, 2] == x[0, 2] and not biased[0, 2]                            # no entry: the bits as they were
    assert f[1] == -np.inf                                                    # a -inf bias bans
    assert np.isnan(f[3]) and np.isnan(f[4])                                  # NaN + 1 and inf + -inf
    assert y[0, 0] == round_to(np.float32(1.0) + np.float32(1e-4), dtype)     # one fp32 add, one rounding
    if dtype == "fp16":
        assert f[0] == np.float16(1.0) and f[7] == np.inf                     # 1 + 1e-4 rounds back to 1; 100 + 7e4 overflows
        assert f[6] == np.float32(np.float16(np.float32(0.5) + np.float32(0.1)))
    if dtype == "fp32":
        assert f[0] == np.float32(1.0) + np.float32(1e-4) and f[7] == np.float32(70100.0)
    assert biased[0].tolist() == [True, True, False, True, True, False, True, True]


def test_oracle_keeps_unbiased_nan_payloads_and_bf16_rounds_to_nearest_even():
    x = np.array([[0x7E01, 0xFE42, 0x3C00]], np.uint16)                       # two fp16 NaNs with payloads, 1.0
    y, _ = constrain(x, "fp16", np.array([[-1]], np.int32))
    assert np.array_equal(y, x)
    # bf16: 1 + 2^-8 is a tie between 1 and 1 + 2^-7: to even (1); 1 + 3 * 2^-8 rounds up to 1 + 2^-6
    assert round_to(np.float32(1 + 2 ** -8), "bf16") == 0x3F80
    assert round_to(np.float32(1 + 3 * 2 ** -8), "bf16") == 0x3F82
    assert round_to(np.float32(3.397e38), "bf16") == 0x7F80                   # a finite fp32 past bf16's max rounds to +inf
    assert to_f32(np.array([0xFF80], np.uint16), "bf16")[0] == -np.inf


def test_oracle_min_p_kept_set():
    p = np.array([[0.5, 0.25, 0.125, 0.125, 0.0], [0.2, 0.2, 0.2, 0.2, 0.2]], np.float32)
    base = np.ones_like(p, bool)
    np.testing.assert_array_equal(min_p_kept(p, base, [0.5, 1.0]), [[1, 1, 0, 0, 0], [1, 1, 1, 1, 1]])   # p == bound is kept
    np.testing.assert_array_equal(min_p_kept(p, base, [0.0, 0.0]), [[1, 1, 1, 1, 1], [1, 1, 1, 1, 1]])
    np.testing.assert_array_equal(min_p_kept(p, base, [2.0, -1.0]), [[1, 0, 0, 0, 0], [1, 1, 1, 1, 1]])  # clamped to [0, 1]
    base[0, 0] = False
    assert not min_p_kept(p, base, [0.9, 0.0])[0].any()                     # an intersection, not a new set


# ---------------------------------------------------------------------------------------------------- the step
def test_decode_step_rejects_constraints_it_cannot_apply():
    with pytest.raises(ValueError, match="tp_size 1"):
        DecodeStep(TINY, 4, 40, None, token_bitmask=True, tp_size=2)
    with pytest.raises(ValueError, match="tp_size 1"):
        DecodeStep(TINY, 4, 40, None, logit_bias_capacity=16, tp_size=2)
    with pytest.raises(ValueError, match="logit_bias_capacity"):
        DecodeStep(TINY, 4, 40, None, logit_bias_capacity=-1)
    for bad in (1.5, -0.1, [0.0, 0.2, 1.1, 0.0]):
        with pytest.raises(ValueError, match="min_p"):
            DecodeStep(TINY, 4, 40, None, sampling=SamplingParams(min_p=bad))
    assert SamplingParams().has_min_p() is False and SamplingParams(min_p=[0.0, 0.0]).has_min_p() is False
    assert SamplingParams(min_p=[0.0, 0.1]).has_min_p() and SamplingParams(min_p=0.05).has_min_p()


def _host_step(R=3, V=100, cap=4, mask=True):
    """A DecodeStep's constraint state with host tensors standing in for the device buffers."""
    s = DecodeStep.__new__(DecodeStep)
    s.B, s.q_len, s.vocab = R, 1, V
    if mask:
        s.bitmask_h = torch.full((R, (V + 31) // 32), -1, dtype=torch.int32)
        s.bitmask = torch.zeros_like(s.bitmask_h)
    if cap:
        s.bias_h = (torch.zeros(R + 1, dtype=torch.int32), torch.zeros(cap, dtype=torch.int32), torch.zeros(cap))
        s.bias = tuple(torch.zeros_like(t) for t in s.bias_h)
    return s


def test_set_constraints_validates_and_fills_the_buffers():
    s = _host_step()
    m = np.arange(12, dtype=np.int32).reshape(3, 4)
    s.set_constraints(bitmask=m, logit_bias=[{1: 2.0}, {}, {7: -1.0, 99: 3.0}])
    assert s.bitmask.numpy().tolist() == m.tolist()
    assert s.bias[0].tolist() == [0, 1, 1, 3] and s.bias[1][:3].tolist() == [1, 7, 99] and s.bias[2][:3].tolist() == [2.0, -1.0, 3.0]
    s.set_constraints()                                                       # back to unconstrained
    assert (s.bitmask == -1).all() and s.bias[0].tolist() == [0, 0, 0, 0]
    for bad in (m[:2], m.astype(np.int64), np.zeros((3, 5), np.int32)):
        with pytest.raises(ValueError, match="bitmask must be host int32"):
            s.set_constraints(bitmask=bad)
    with pytest.raises(ValueError, match="one mapping per logits row"):
        s.set_constraints(logit_bias=[{}, {}])
    with pytest.raises(ValueError, match="exceed logit_bias_capacity 4"):
        s.set_constraints(logit_bias=[{1: 1.0, 2: 1.0}, {3: 1.0}, {4: 1.0, 5: 1.0}])
    with pytest.raises(ValueError, match="outside"):
        s.set_constraints(logit_bias=[{}, {100: 1.0}, {}])
    with pytest.raises(ValueError, match="not a number"):
        s.set_constraints(logit_bias=[{}, {1: float("nan")}, {}])
    with pytest.raises(ValueError, match="without token_bitmask"):
        _host_step(mask=False).set_constraints(bitmask=m)
    with pytest.raises(ValueError, match="without logit_bias_capacity"):
        _host_step(cap=0).set_constraints(logit_bias=[{}, {}, {}])
