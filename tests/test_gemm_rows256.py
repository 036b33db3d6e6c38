"""Host side of the 256-row weight-only GEMM, without a GPU: the workspace the library asks for at 1..256 rows, the row
limits of b200_wo_gemm and of the decode step's modes (max_rows), all checked before any CUDA call."""
import ctypes

import pytest

from rtp_llm_b200 import _lib
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams
from tests import program_chains as pc

SHAPES = [(4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096), (4096, 128256), (1024, 384), (384, 200)]   # (K, N)


def _plan(K, N):
    ns, kbp = ctypes.c_int(), ctypes.c_int()
    assert _lib.load().b200_plan_gemm_split(K, N, ctypes.byref(ns), ctypes.byref(kbp)) == 0
    return ns.value


def _partials(n_tiles, S, bpad):
    return n_tiles * S * bpad * 128 * 4 if S > 1 else 0


@pytest.mark.parametrize("K,N", SHAPES)
def test_workspace_bytes_at_1_to_256_rows(K, N):
    """129..256 rows: the counters plus n_tiles * S * 256 * 128 fp32 partials of the split plan's S (the persistent kernel
    holds no GEMM at batch pad 256). 1..128 rows: the plain plan's or the persistent plan's partials, whichever is larger,
    as before."""
    lib = _lib.load()
    n_tiles, S = -(-N // 128), _plan(K, N)
    for B in (129, 130, 192, 255, 256):
        assert lib.b200_wo_gemm_workspace_bytes(B, N, K) == pc.SEM_BYTES + _partials(n_tiles, S, 256), B
    for B in (1, 16, 17, 33, 64, 65, 128):
        bpad = pc.bpad_of(B)
        per = pc.sk_plan(n_tiles, K // 128, 2 * pc.SMS, bpad)
        persistent = n_tiles * (K // 128 // per) * bpad * 128 * 4 if per < K // 128 else 0
        assert lib.b200_wo_gemm_workspace_bytes(B, N, K) == pc.SEM_BYTES + max(_partials(n_tiles, S, bpad), persistent), B
    assert lib.b200_wo_gemm_workspace_bytes(257, N, K) == 0


def test_257_rows_are_refused_on_the_host():
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.b200_wo_gemm(_lib.B200_FMT_INT4, 0, p, 257, 128, 128, p, None, None, p, p, 4096, 0, None) == -1
    assert b"1..256" in lib.b200_last_error()
    regions = (ctypes.c_void_p * 2)(p, p)
    assert lib.b200_wo_gemm_rs(_lib.B200_FMT_INT4, 0, p, 129, 128, 128, p, None, None, p, p, 4096, 0, regions, 1 << 20, 0, 2,
                               None) == -1
    assert b"1..128" in lib.b200_last_error()


def test_decode_step_rejects_more_than_256_rows_and_tp_above_128():
    with pytest.raises(ValueError, match="256"):
        DecodeStep(TINY, 257, 40, None)
    with pytest.raises(ValueError, match="tp_size"):
        DecodeStep(TINY, 129, 40, None, tp_size=2)


def test_max_rows_widens_the_verification_tree_beam_and_sampling_modes_to_256():
    """By default these modes keep their 128-row limit (the existing rejection tests); max_rows=256 moves the limit to 256
    rows, the GEMM's, with the same rejection beyond it, and only in 1..256."""
    sp = SamplingParams(top_k=50, top_p=0.9)
    for kw in (dict(q_len=4), dict(q_len=4, tree=[-1, 0, 0, 1]), dict(beam_width=4), dict(sampling=sp, q_len=4)):
        with pytest.raises(ValueError, match="<= 256 .max_rows"):
            DecodeStep(TINY, 65, 40, None, max_rows=256, **kw)
        with pytest.raises(ValueError, match="<= 128 .max_rows"):
            DecodeStep(TINY, 33, 40, None, **kw)
    with pytest.raises(ValueError, match="<= 256 .max_rows"):
        DecodeStep(TINY, 257, 40, None, sampling=sp, max_rows=256)
    with pytest.raises(ValueError, match="tp_size"):
        DecodeStep(TINY, 4, 40, None, q_len=2, tp_size=2, max_rows=256)
    for bad in (0, 257):
        with pytest.raises(ValueError, match="max_rows must be in 1..256"):
            DecodeStep(TINY, 4, 40, None, max_rows=bad)
