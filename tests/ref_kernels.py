"""ctypes face of tests/native/libb200_testref.so: deliberately naive CUDA-core kernels over the UN-permuted reference
tensors. Test infrastructure (a second opinion next to the CPU oracle), never part of the product library."""
import ctypes
import os
from ctypes import c_float, c_int, c_uint64, c_void_p

import torch

from rtp_llm_b200._lib import B200_FMT_INT4

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "native", "libb200_testref.so")
_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from rtp_llm_b200 import build as b
            b.build_testref()
        lib = ctypes.CDLL(LIB_PATH)
        lib.b200_ref_paged_decode_attn.restype = c_int
        lib.b200_ref_paged_decode_attn.argtypes = [c_void_p, c_int, c_void_p] + [c_int] * 6 + [c_void_p] * 3 + [c_float, c_void_p]
        lib.b200_ref_dequant_gemm.restype = c_int
        lib.b200_ref_dequant_gemm.argtypes = [c_int, c_int, c_void_p, c_int, c_int, c_int] + [c_void_p] * 3 + [c_int, c_void_p,
                                                                                                        c_void_p, c_void_p]
        lib.b200_ref_pdl_writer.restype = c_int
        lib.b200_ref_pdl_writer.argtypes = [c_void_p, c_int, c_int, c_uint64, c_void_p, c_void_p]
        lib.b200_ref_pdl_probe.restype = c_int
        lib.b200_ref_pdl_probe.argtypes = [c_int] * 5 + [c_void_p, c_void_p]
        lib.b200_ref_pdl_copy.restype = c_int
        lib.b200_ref_pdl_copy.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p]
        _lib = lib
    return _lib


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def ref_paged_decode_attn(q, kv_cache_base, page_list, sequence_lengths, q_scale=1.0):
    P, two, Hkv, T, D = kv_cache_base.shape
    B = q.shape[0]
    Hq = q.numel() // (B * D)
    out = torch.empty((B, Hq * D), dtype=q.dtype, device=q.device)
    rc = load().b200_ref_paged_decode_attn(_p(q), 1 if q.dtype == torch.bfloat16 else 0, _p(out), Hq, Hkv, D, B, page_list.shape[-1], T,
                                           _p(kv_cache_base), _p(page_list), _p(sequence_lengths), q_scale, _stream())
    assert rc == 0, rc
    return out


def ref_dequant_gemm(x, fmt, w, scales=None, zeros_x_scales=None, group=128, bias=None):
    """fmt F16: w [K,N]; INT8: w int8 [K,N] + scales [N]; INT4: w uint8 [K,N/2] + scales/zeros [K/g,N]."""
    B, K = x.shape
    N = w.shape[1] * (2 if fmt == B200_FMT_INT4 else 1)
    out = torch.empty((B, N), dtype=x.dtype, device=x.device)
    rc = load().b200_ref_dequant_gemm(fmt, 1 if x.dtype == torch.bfloat16 else 0, _p(x), B, K, N, _p(w), _p(scales), _p(zeros_x_scales),
                                      group, _p(bias), _p(out), _stream())
    assert rc == 0, rc
    return out


def pdl_writer(copies, n_snap, n_stage, delay_ns, times):
    """The PDL harness's slow predecessor on the current stream: copies int64 [n_snap + n_stage, 3] rows of (source, destination,
    bytes), the snapshot ranges first; times int64 [2] receives %globaltimer before and after the copies."""
    rc = load().b200_ref_pdl_writer(_p(copies), n_snap, n_stage, delay_ns, _p(times), _stream())
    assert rc == 0, rc


def pdl_probe(grid_x, grid_y, threads, smem, cluster_x, entry):
    """A PDL-attributed kernel of that shape whose CTAs store %globaltimer at entry into entry int64 [grid_x * grid_y]."""
    rc = load().b200_ref_pdl_probe(grid_x, grid_y, threads, smem, cluster_x, _p(entry), _stream())
    assert rc == 0, rc


def pdl_copy(x, out, mode):
    """The harness's control (int32 x -> out, PDL attribute): 0 waits first, 1 loads x before the wait, 2 stores before it."""
    rc = load().b200_ref_pdl_copy(_p(x), _p(out), x.numel(), mode, _stream())
    assert rc == 0, rc
