"""Python face of the CPU oracle (TEST INFRASTRUCTURE ONLY -- see decode_oracle.c header).

Two layers:
  * ctypes bindings to oracle/liboracle.so (the C restatement, also the timed CPU arm), and
  * small pure-numpy restatements of the same functions used to cross-check the C code on tiny cases.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may import this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB: Optional[ctypes.CDLL] = None


def build() -> str:
    """Compile oracle/liboracle.so (gcc, OpenMP). Building the checker is not using it."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    return os.path.join(_HERE, "liboracle.so")


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build()
        _LIB = ctypes.CDLL(path)
        _LIB.oracle_num_threads.restype = ctypes.c_int
        _LIB.oracle_paged_attn_plan.restype = ctypes.c_int
    return _LIB


def _p(a: np.ndarray):
    assert a.flags["C_CONTIGUOUS"], "oracle expects contiguous arrays"
    return a.ctypes.data_as(ctypes.c_void_p)


def num_threads() -> int:
    return int(lib().oracle_num_threads())


# ----------------------------------------------------------------------------------------------
# 16-bit helpers: tensors cross the oracle boundary as uint16 bit patterns
# ----------------------------------------------------------------------------------------------
def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    lsb = (u >> 16) & 1
    return ((u + 0x7FFF + lsb) >> 16).astype(np.uint16)


def bf16_bits_to_f32(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << 16).view(np.float32)


def to_bits(x: np.ndarray, is_bf16: bool) -> np.ndarray:
    if x.dtype == np.uint16:
        return np.ascontiguousarray(x)
    if is_bf16:
        return f32_to_bf16_bits(x)
    return np.ascontiguousarray(x.astype(np.float16)).view(np.uint16)


def from_bits(b: np.ndarray, is_bf16: bool) -> np.ndarray:
    return bf16_bits_to_f32(b) if is_bf16 else b.view(np.float16).astype(np.float32)


# ----------------------------------------------------------------------------------------------
# Indexing
# ----------------------------------------------------------------------------------------------
def convert_block_table(block_ids: np.ndarray) -> np.ndarray:
    """kv_cache_kernels.cu:49-63. [B,M] int32 -> [B,1,2,M] int32 (K page 2*id, V page 2*id+1)."""
    block_ids = np.ascontiguousarray(block_ids, dtype=np.int32)
    B, M = block_ids.shape
    out = np.empty((B, 1, 2, M), dtype=np.int32)
    lib().oracle_convert_block_table(_p(out), _p(block_ids), B, M)
    return out


def convert_block_table_np(block_ids: np.ndarray) -> np.ndarray:
    b = np.asarray(block_ids, dtype=np.int32)
    return np.stack([b * 2, b * 2 + 1], axis=1)[:, None, :, :].astype(np.int32)


def paged_attn_plan(sequence_lengths, block_ids, tokens_per_block, input_lengths=None, prefix_lengths=None):
    """mha_paged_attn_plan.cu:28-97. Returns dict of last_page_len, page_indptr, page_indice, batch_indice, positions."""
    B = len(sequence_lengths) if prefix_lengths is None else len(prefix_lengths)
    block_ids = np.ascontiguousarray(block_ids, dtype=np.int32)
    M = block_ids.shape[1]
    seq = np.ascontiguousarray(sequence_lengths, dtype=np.int32) if sequence_lengths is not None else None
    inl = np.ascontiguousarray(input_lengths, dtype=np.int32) if input_lengths is not None else None
    pre = np.ascontiguousarray(prefix_lengths, dtype=np.int32) if prefix_lengths is not None else None
    ntok = int(inl.sum()) if pre is not None else B
    last = np.zeros(B, np.int32)
    indptr = np.zeros(B + 1, np.int32)
    indice = np.zeros(B * M, np.int32)
    bidx = np.zeros(max(ntok, 1), np.int32)
    pos = np.zeros(max(ntok, 1), np.int32)
    total = lib().oracle_paged_attn_plan(
        _p(inl) if inl is not None else None,
        _p(seq) if seq is not None else None,
        _p(pre) if pre is not None else None,
        _p(block_ids), B, M, int(tokens_per_block), _p(last), _p(indptr), _p(indice), _p(bidx), _p(pos))
    return dict(last_page_len=last, page_indptr=indptr, page_indice=indice[:total], batch_indice=bidx[:ntok],
                positions=pos[:ntok])


# ----------------------------------------------------------------------------------------------
# Paged decode attention
# ----------------------------------------------------------------------------------------------
def paged_decode_attn(q_bits, kv_pool_bits, page_list, sequence_lengths, head_num, kv_head_num, head_dim,
                      tokens_per_block, is_bf16=False, q_scale=1.0) -> np.ndarray:
    """q [B,Hq,D] bits, kv_pool [P,2,Hkv,T,D] bits, page_list [B,1,2,M] int32, sequence_lengths [B] (past len).
    Returns out bits [B, Hq*D]."""
    q_bits = np.ascontiguousarray(q_bits, dtype=np.uint16)
    kv_pool_bits = np.ascontiguousarray(kv_pool_bits, dtype=np.uint16)
    page_list = np.ascontiguousarray(page_list, dtype=np.int32)
    seq = np.ascontiguousarray(sequence_lengths, dtype=np.int32)
    B = q_bits.shape[0]
    M = page_list.shape[-1]
    out = np.empty((B, head_num * head_dim), dtype=np.uint16)
    lib().oracle_paged_decode_attn(_p(q_bits), int(is_bf16), _p(out), head_num, kv_head_num, head_dim, B, M,
                                   tokens_per_block, _p(kv_pool_bits), _p(page_list), _p(seq),
                                   ctypes.c_float(q_scale))
    return out


def paged_decode_attn_np(q, kv_pool, block_ids, sequence_lengths, tokens_per_block, q_scale=1.0, with_abs=False):
    """Float64 restatement with no P rounding: the reference the attention error budget is measured from.

    q [B,Hq,D], or [B,q_len,Hq,D] for several query tokens per sequence (query j sees positions 0 .. seq[b] + j);
    kv_pool [P,2,Hkv,T,D] float; block_ids [B,M]. Returns out [B, Hq*D] (or [B, q_len, Hq*D]); with_abs=True returns
    (out, E), where E = sum_t p_t |v_t| / sum_t p_t, of the same shape, is the size of the terms the output averages
    (see attn_error_budget)."""
    multi = q.ndim == 4
    q4 = q if multi else q[:, None]
    B, QL, Hq, D = q4.shape
    Hkv = kv_pool.shape[2]
    g = Hq // Hkv
    T = tokens_per_block
    out = np.zeros((B, QL, Hq, D), np.float64)
    E = np.zeros_like(out)
    for b in range(B):
        L = int(sequence_lengths[b]) + QL
        pages = np.asarray(block_ids[b][: (L + T - 1) // T], np.int64)
        kv = np.asarray(kv_pool[pages], np.float64)                               # [pages, 2, Hkv, T, D]
        k = kv[:, 0].transpose(1, 0, 2, 3).reshape(Hkv, -1, D)[:, :L]            # [Hkv, L, D]
        v = kv[:, 1].transpose(1, 0, 2, 3).reshape(Hkv, -1, D)[:, :L]
        qh = np.asarray(q4[b], np.float64).reshape(QL, Hkv, g, D).transpose(1, 0, 2, 3).reshape(Hkv, QL * g, D)
        s = (qh @ k.transpose(0, 2, 1)) * (q_scale / np.sqrt(D))                  # [Hkv, QL*g, L]
        seen = np.arange(L)[None, :] <= (L - QL + np.arange(QL))[:, None]         # [QL, L]
        s = np.where(np.repeat(seen, g, axis=0)[None], s, -np.inf)
        p = np.exp(s - s.max(-1, keepdims=True))
        den = p.sum(-1, keepdims=True)
        o, e = (p @ v) / den, (p @ np.abs(v)) / den                               # [Hkv, QL*g, D]
        out[b] = o.reshape(Hkv, QL, g, D).transpose(1, 0, 2, 3).reshape(QL, Hq, D)
        E[b] = e.reshape(Hkv, QL, g, D).transpose(1, 0, 2, 3).reshape(QL, Hq, D)
    shape = (B, QL, Hq * D) if multi else (B, Hq * D)
    return (out.reshape(shape), E.reshape(shape)) if with_abs else out.reshape(shape)


def ulp(x: np.ndarray, is_bf16: bool) -> np.ndarray:
    """Spacing of fp16 / bf16 numbers at |x| (subnormal spacing below the smallest normal)."""
    mant, emin = (7, -126) if is_bf16 else (10, -14)
    e = np.floor(np.log2(np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** emin)))
    return 2.0 ** (e - mant)


def attn_error_budget(ref: np.ndarray, E: np.ndarray, is_bf16: bool) -> np.ndarray:
    """Per-element bound on |got - ref| for a correct paged decode attention kernel in T = fp16 / bf16, against the float64
    reference (ref, E) of paged_decode_attn_np:  ulp_T(ref) + u_T * (E + |ref|),  u = 2^-11 (fp16) or 2^-8 (bf16).

    Why: the kernel computes O = sum_t P_t v_t / l with l = sum_t p_t kept in fp32, and P_t = p_t rounded once to T as
    the A operand of the PV product. Rounding to nearest moves each p_t by at most u * p_t (p_t in T's normal range, which
    holds for every p_t that matters at the scores these tests draw), so the numerator moves by
    at most u * sum_t p_t |v_t| and O by at most u * E. The fp32 work (scores, exp2, the row sum, the split merges) adds
    errors of order 2^-24 per operation, far below u; u * |ref| covers it. The one final rounding of O to T costs half
    an ulp_T(ref), and ulp_T(ref) leaves room for the fp32 terms near zero. The bound does not depend on the sequence
    length, so a dropped token, tile or split, whose effect on the output shrinks like 1/L, still exceeds it where a
    fixed rtol/atol of 1e-2 stops seeing it. The C oracle, which rounds P as the kernel does, stays near 0.12 of it."""
    u = 2.0 ** -8 if is_bf16 else 2.0 ** -11
    return ulp(ref, is_bf16) + u * (np.asarray(E, np.float64) + np.abs(ref))


# ----------------------------------------------------------------------------------------------
# Weight-only GEMM: float64 reference, error budget and exact rounding
# ----------------------------------------------------------------------------------------------
def round_t(x, is_bf16: bool) -> np.ndarray:
    """float64 -> the nearest fp16 / bf16 value, ties to even, rounded ONCE (returned as float64). Subnormals are kept,
    values past the largest finite number by half an ulp or more become +-inf, NaN stays NaN. numpy's float64 -> float16
    cast is the same single rounding; a float64 -> float32 -> bf16 chain rounds twice and can differ at ties."""
    mant, emin, emax = (7, -126, 127) if is_bf16 else (10, -14, 15)
    x = np.asarray(x, np.float64)
    _, e = np.frexp(x)                                         # x = m * 2^e, 0.5 <= |m| < 1: floor(log2 |x|) = e - 1, exactly
    q = np.ldexp(1.0, np.maximum(e - 1, emin) - mant)          # the spacing of T at |x|
    r = np.round(x / q) * q                                    # x / q is exact (q a power of two); np.round ties to even
    r = np.where(np.abs(r) > (2.0 - 2.0 ** -mant) * 2.0 ** emax, np.copysign(np.inf, x), r)
    return np.where(np.isfinite(x), r, x)


def f64_to_bits(x, is_bf16: bool) -> np.ndarray:
    """float64 -> fp16 / bf16 bit patterns (uint16) with the one rounding of round_t."""
    r = round_t(x, is_bf16)
    if is_bf16:
        return (r.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)   # r is a bf16 value: the float32 cast is exact
    return r.astype(np.float16).view(np.uint16)


def _vals(a, is_bf16: bool) -> np.ndarray:
    """fp16 / bf16 values as float64, from uint16 bit patterns or from any float array that already holds T values."""
    a = np.asarray(a)
    return from_bits(a, is_bf16).astype(np.float64) if a.dtype == np.uint16 else a.astype(np.float64)


def dequant_exact(fmt: str, weight, scales=None, zeros_x_scales=None, group: int = 128, is_bf16=False) -> np.ndarray:
    """The weight W' [K,N] the GEMM's tensor cores multiply, in float64 (every value exactly a T value):
      * int4 (group 128 / 64 / 32) and int8g: W' = round_T(q_s * s + zs), ONE rounding, as hfma2(q_s, s, zs) in the kernel
        (Dequant4, dequant_half). q_s (<= 8 bits) * s (<= 11) is exact in float64, and so is the sum with zs at any exponent
        gap below 2^30, so the only rounding is round_t's. The group of row k is k // group.
      * int8 per-column: W' = q_s, exact; the column scale is the epilogue's (gemm_np's cscale).
      * f16: W' = W.
    weight: int4 uint8 [K,N/2] (low nibble = even column); int8 / int8g int8 [K,N]; f16 the values or their bits.
    scales / zeros_x_scales [K/group, N]: the values (as float) or their uint16 bits. Unlike dequant_np, nothing passes through
    float32 on the way."""
    if fmt == "f16":
        return _vals(weight, is_bf16)
    if fmt == "int8":
        return np.asarray(weight).astype(np.float64)
    if fmt not in ("int4", "int8g"):
        raise ValueError(fmt)
    q = unpack_int4_signed(weight) if fmt == "int4" else np.asarray(weight)
    s = np.repeat(_vals(scales, is_bf16), group, axis=0)
    z = np.repeat(_vals(zeros_x_scales, is_bf16), group, axis=0)
    return round_t(q.astype(np.float64) * s + z, is_bf16)


def gemm_np(x, w_deq, cscale=None, bias=None) -> Tuple[np.ndarray, np.ndarray]:
    """Float64 Y = (X . W') * cscale + bias and the size of its terms A = (|X| . |W'|) * |cscale| + |bias| (both [B,N]).
    x [B,K], w_deq [K,N] (dequant_exact), cscale / bias [N] or None; all float values (T values in practice)."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w_deq, np.float64)
    ref, A = x @ w, np.abs(x) @ np.abs(w)
    if cscale is not None:
        c = np.asarray(cscale, np.float64)[None, :]
        ref, A = ref * c, A * np.abs(c)
    if bias is not None:
        b = np.asarray(bias, np.float64)[None, :]
        ref, A = ref + b, A + np.abs(b)
    return ref, A


def gemm_fp32_error(A: np.ndarray, K: int, nsplit: int = 1) -> np.ndarray:
    """Bound on |v - ref| for the fp32 value v the GEMM's epilogue holds before its final rounding to T (see
    gemm_error_budget): 2^-24 * (272 * kbp + nsplit) * A, kbp = the k-blocks of the longest split."""
    kb = -(-int(K) // 128)
    kbp = -(-kb // max(int(nsplit), 1))
    return 2.0 ** -24 * (272 * kbp + nsplit) * np.asarray(A, np.float64)


def gemm_error_budget(ref: np.ndarray, A: np.ndarray, K: int, nsplit: int, is_bf16: bool) -> np.ndarray:
    """Per-element bound on |y - ref| for a correct weight-only GEMM in T = fp16 / bf16, against gemm_np's (ref, A):
    ulp_T(ref) + c * A,  c = 2^-24 * (272 * kbp + nsplit),  kbp = ceil(ceil(K / 128) / nsplit).

    Why: every product x_k * W'_k is exact in fp32 (two T significands, <= 22 bits). A split of kbp k-blocks accumulates them
    in 8 * kbp tensor-core k16 steps, each adding 16 products to the fp32 accumulator. How the hardware rounds inside that
    sum is not documented, so the bound assumes the worst of a 24-bit adder without guard bits: the 17 addends (the
    accumulator and 16 products) are aligned to the largest exponent E and each of the 16 shifted ones is truncated to a
    multiple of 2^(E-23), losing up to 2^(E-23) <= 2^-23 * max|addend| each; the sum is then normalised to 24 bits by
    truncation, losing up to another 2^-23 of its magnitude. Every addend and every running sum is at most A (the sum of
    |terms|), so one step loses at most 17 * 2^-23 * A = 34 * 2^-24 * A, and the chain of 8 * kbp steps 272 * kbp * 2^-24 * A.
    The nsplit fp32 partials are merged in a fixed order with round-to-nearest adds (nsplit - 1 of them, 2^-24 * A each),
    and the epilogue's fmaf(acc, cscale, bias) rounds once more (2^-24 * A). The one final rounding to T costs half an
    ulp_T; ulp_T(ref) leaves room for the value crossing a binade. A call whose split is not known may pass nsplit = 1:
    that bound is the loosest for any split <= 16. The one assumption is that the adder keeps at least fp32's 24 bits
    at the largest addend's exponent; a narrower window is not an fp32 accumulation.

    The bound grows with K because it is a worst case; a kernel rounding to nearest and summing random-signed terms stays
    far below it. gemm_rounded_fractions is the sharper check for that regime. Measured on an H100 80GB HBM3 (700 W power
    limit): see DESIGN section 4 for the worst err/budget per path and dtype; everywhere it is below 0.5 -- the final
    rounding's half ulp, with the fp32 error far below c * A."""
    return ulp(ref, is_bf16) + gemm_fp32_error(A, K, nsplit)


def _ordinal(bits: np.ndarray) -> np.ndarray:
    """fp16 / bf16 bit patterns -> integers in the order of their values, adjacent values one apart (+0 and -0 both 0)."""
    b = np.asarray(bits, np.uint16).astype(np.int32)
    mag = b & 0x7FFF
    return np.where(b & 0x8000, -mag, mag)


# Thresholds of gemm_rounded_fractions for random data (see its docstring for the measured values they leave room below).
GEMM_MIN_ROUNDED = 0.9
GEMM_MIN_WITHIN_ONE = 0.99


def gemm_rounded_fractions(got, ref, is_bf16: bool) -> Tuple[float, float]:
    """(fraction of outputs equal to round_T(ref), fraction at most one T step away from it). got: the kernel's output as
    T values or uint16 bits; ref: gemm_np's float64 result.

    An fp32 kernel's accumulation error is small next to ulp_T(y) for all but the outputs much smaller than their terms
    (|y| << A), so it rounds almost every output correctly and hardly any by more than one step. A kernel that rounds its
    split partials or W' twice adds an error of a good fraction of an ulp_T to most outputs, which the worst-case budget
    still allows at large K, and drops well below both thresholds. At the Llama-3-8B w2 shape (B 32, K 14336, INT4,
    tests/test_gemm_budget.py) a simulated round-to-nearest fp32 kernel gives 0.998 / 0.9998 (fp16, unsplit) and
    0.9996 / 0.99998 (bf16); the two double-rounding mutants give 0.56-0.59 / 0.86-0.88. On an H100 80GB HBM3 (700 W
    power limit), over the 289 random-data GEMM cases of the suite, the kernels gave at least 0.980 / 0.9974. Thresholds
    GEMM_MIN_ROUNDED = 0.9 / GEMM_MIN_WITHIN_ONE = 0.99 leave room below that and stay above the mutants."""
    g = np.asarray(got)
    gb = g if g.dtype == np.uint16 else f64_to_bits(g.astype(np.float64), is_bf16)
    rb = f64_to_bits(ref, is_bf16)
    d = np.abs(_ordinal(gb) - _ordinal(rb))
    bad = np.isnan(from_bits(gb, is_bf16))
    return float(((d == 0) & ~bad).mean()), float(((d <= 1) & ~bad).mean())


def silu_mul_np(g: np.ndarray, u: np.ndarray) -> np.ndarray:
    """Float64 silu(g) * u."""
    return g / (1.0 + np.exp(-g)) * u


def silu_mul_budget(g, Ag, u, Au, K: int, nsplit: int, is_bf16: bool) -> np.ndarray:
    """Bound on |y - silu(g) u| for the fused SiLU*mul epilogue, from the float64 gate / up (g, Ag), (u, Au) of gemm_np. The
    kernel evaluates __fdividef(g, 1 + __expf(-g)) * u on its fp32 g, u (each within e = gemm_fp32_error of the reference)
    and rounds once to T. |silu'| <= 1.1 everywhere, so the inputs' errors move the result by at most
    1.1 e_g (|u| + e_u) + |silu(g)| e_u; __expf is within 2 + 1.16 |g| fp32 ulps and the divide within 2 ulps, the multiply
    half an ulp, so the evaluation adds at most 2^-23 (6 + 2 |g|) |result|; the final rounding is within ulp_T."""
    g, u = np.asarray(g, np.float64), np.asarray(u, np.float64)
    eg, eu = gemm_fp32_error(Ag, K, nsplit), gemm_fp32_error(Au, K, nsplit)
    ref = silu_mul_np(g, u)
    sg = g / (1.0 + np.exp(-g))
    return ulp(ref, is_bf16) + 1.1 * eg * (np.abs(u) + eu) + np.abs(sg) * eu + 2.0 ** -23 * (6 + 2 * np.abs(g)) * np.abs(ref)


# ----------------------------------------------------------------------------------------------
# Glue ops: float64 references and error budgets (RMSNorm, QK-RMSNorm, RoPE); SiLU*mul reuses silu_mul_np / _budget
# ----------------------------------------------------------------------------------------------
def rmsnorm_np(x, residual, gamma, eps, bias=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Float64 RMSNorm of the rows of x (+ residual), flashinfer's fused-add contract (DESIGN section 3.3): s = x + r exact,
    y = s * g / sqrt(mean(s^2) + eps) (+ bias), and the stored residual round_T(s) is round_t(s) by the caller.
    x, residual [rows, n] (residual may be None), gamma / bias [n]: T values as floats (or anything float). eps is taken
    as the fp32 value the kernels receive. Returns (y, s, A): A = |s * g / rms| + |bias|, the size of the terms of y that
    norm_error_budget scales. QK-RMSNorm is this per head, with the bias added before the one rounding to T."""
    s = np.asarray(x, np.float64)
    if residual is not None:
        s = s + np.asarray(residual, np.float64)
    inv = 1.0 / np.sqrt(np.mean(s * s, axis=-1, keepdims=True) + float(np.float32(eps)))
    y = s * inv * np.asarray(gamma, np.float64)
    A = np.abs(y)
    if bias is not None:
        b = np.asarray(bias, np.float64)
        y, A = y + b, A + np.abs(b)
    return y, s, A


def norm_chain(hidden: int, threads: int) -> int:
    """The longest fp32 add chain of a norm kernel's sum of squares: the per-thread fmaf chain (8 elements per 16-byte
    vector, ceil(hidden / 8 / threads) vectors) plus 16 for the warp butterfly and the cross-warp sum (5 + at most 8 adds in
    the persistent kernel, 5 + 5 in the stand-alone one)."""
    return 8 * (-(-hidden // (8 * threads))) + 16


def norm_error_budget(ref: np.ndarray, A: np.ndarray, chain: int, is_bf16: bool) -> np.ndarray:
    """Per-element bound on |y - ref| for an RMSNorm kernel in T = fp16 / bf16 against rmsnorm_np's (ref, A):
    ulp_T(ref) + 2^-24 * (chain / 2 + 12) * A, chain = norm_chain(...) (QK-RMSNorm: head_dim / 32 + 5).

    Why (u = 2^-24, the relative error of one fp32 rounding to nearest): s = x + r rounds once in fp32 (u |s|; exact
    unless the two exponents are more than 13 apart). The sum of squares is a tree of nonnegative terms whose deepest path
    is `chain` roundings (each fmaf of the per-thread chain rounds once, each butterfly or cross-warp add once), so it is
    within chain * u of the exact sum, relatively. The mean (a division by hidden) and + eps round once each; rsqrtf is
    within 2 ulp (CUDA C Programming Guide, table of single-precision functions), 4 u relatively; the square root halves
    the relative error of its argument, so 1 / rms is within ((chain + 2) / 2 + 4 + 1) u. The two products s * inv * g round
    once each (2 u), the optional bias add once more (u relative to A). In all, (chain / 2 + 9) u of A; 12 leaves room for
    the first-order terms dropped. The one final rounding to T is half an ulp_T; ulp_T(ref) leaves room for the value
    crossing a binade. eps is inside the square root, so a row whose mean square is near eps is no harder: the bound is
    relative to the output, and a kernel that adds eps after the square root misses it by far on such rows."""
    return ulp(ref, is_bf16) + 2.0 ** -24 * (chain / 2 + 12) * np.asarray(A, np.float64)


# Thresholds of gemm_rounded_fractions for the glue ops on random data (correctly rounded, within one T step), set below
# what the kernels gave on an H100 80GB HBM3 (700 W power limit) over the cases of tests/test_gpu_glue_exact.py and above
# the CPU mutants of tests/test_glue_budget.py.
# Norms (stand-alone, persistent kernel, QK-RMSNorm): at least 0.99951 / 1.0 measured; rounding y twice or s before the
# variance gives 0.74-0.80 correctly rounded.
NORM_MIN_ROUNDED = 0.99
NORM_MIN_WITHIN_ONE = 0.9999
# SiLU*mul (one fp32 evaluation of a few ulps, rounded once): at least 0.99991 / 1.0 measured.
SILU_MIN_ROUNDED = 0.99
SILU_MIN_WITHIN_ONE = 0.9999
# RoPE, over the outputs whose fp32 error bound is below an eighth of ulp_T (rope_fraction_mask: the short positions, where
# the angle is nearly exact): at least 0.99898 / 1.0 measured; a bias added without rounding it to T first gives 0.79-0.81
# / 0.978-0.987 there.
ROPE_MIN_ROUNDED = 0.99
ROPE_MIN_WITHIN_ONE = 0.9999

ROPE_PI32 = float(np.float32(3.141592654))       # the kernels' fp32 pi (Yarn's correction range, Llama3's wavelength)


def yarn_ramp_bounds(cfg) -> Tuple[float, float]:
    """Yarn's ramp bounds (lo, hi) as aux_kernels.cuh rope_coef computes them: from (int)base, floor / ceil to integers,
    clamped to [0, dim - 1], hi nudged by 0.001 when they meet. They do not depend on the position."""
    dim, mp = int(cfg["dim"]), float(np.float32(cfg["max_pos"]))
    t1 = 2.0 * np.log(float(int(np.float32(cfg["base"]))))
    f1, f2 = float(np.float32(cfg["factor1"])), float(np.float32(cfg["factor2"]))
    low = int(np.floor(dim * np.log(mp / (f2 * 2 * ROPE_PI32)) / t1))
    high = int(np.ceil(dim * np.log(mp / (f1 * 2 * ROPE_PI32)) / t1))
    lo, hi = float(max(low, 0)), float(min(high, dim - 1))
    if lo == hi:
        hi += 0.001
    return lo, hi


def rope_angle_np(cfg, zid, pos, seq_len=None) -> Tuple[np.ndarray, float, np.ndarray]:
    """Float64 angle of channel pair zid / 2 (zid = 2i) at integer position pos, and the coefficient scale, for the rope
    contract of b200_rope_append_ex (aux_kernels.cuh rope_coef, DESIGN section 4), and dA, a bound on how far the kernel's
    fp32 angle may be from it. cfg: the RopeConfig fields (its floats taken as the fp32 values the kernel holds); the plain
    kernels' angle is rope_plain_angle_np. seq_len defaults to pos + 1 (the NTK styles' step uses it; a test may move it).
    Returns (a, sc, dA), a / dA broadcast over zid and pos.

    dA, in units of u = 2^-24 times |a|: powf is within 4 ulp (8 u) and its exponent zid / dim rounds once (u times
    |log(base')| times zid / dim); the division pos / powf rounds once; every later fp32 step (/ scale, Yarn's blend of
    three roundings, Llama3's smooth factor, whose relative error ~6 u * (max_pos / wavelen + factor1) / (factor2 - factor1)
    moves a by that times |a - a / scale| <= |a|) adds its own. For the NTK styles past max_pos the rescaled base' =
    base * powf(X, dim / (dim - 2)) carries powf's 8 u, the exponent's rounding times |log X| and X's own three or four
    roundings amplified by dim / (dim - 2) <= 2: bounded by 64 u here, and it reaches a through the exponent zid / dim <= 1."""
    c = {k: float(np.float32(v)) if isinstance(v, float) else v for k, v in cfg.items()}
    style, dim, mp = int(c["style"]), int(c["dim"]), int(c["max_pos"])
    zid = np.asarray(zid, np.float64)
    pos = np.asarray(pos, np.float64)
    sl = pos + 1 if seq_len is None else np.asarray(seq_len, np.float64)
    base = np.full(np.broadcast(zid, pos).shape, c["base"])
    eb = np.zeros_like(base)
    if style == 3:
        X = c["scale"] * sl / mp - (c["scale"] - 1.0)
        step = sl > mp
        base = np.where(step, c["base"] * np.abs(X) ** (dim / (dim - 2.0)), base)
        eb = np.where(step, 64.0, 0.0) + eb
    if style == 4:
        ctx = np.log2(sl / mp) + 1.0
        ntk = np.maximum(2.0 ** np.ceil(ctx) - 1.0, 1.0)
        step = sl > mp
        base = np.where(step, c["base"] * ntk ** (dim / (dim - 2.0)), base)
        eb = np.where(step, 64.0, 0.0) + eb
    t = zid / dim
    a = pos / base ** t
    da = 8.0 + 1.0 + t * eb + t * np.abs(np.log(base)) + 1.0
    sc = 1.0
    if style in (1, 7):
        a = a / c["scale"]
        da = da + 1.0
    elif style == 5:
        lo, hi = yarn_ramp_bounds(c)
        ramp = np.clip((np.floor(zid / 2) - lo) / (hi - lo), 0.0, 1.0)
        mask = (1.0 - ramp) * c["extrapolation_factor"]
        a = (a / c["scale"]) * (1.0 - mask) + a * mask
        da = da + 8.0
        sc = c["mscale"]
    elif style == 6:
        wavelen = np.where(a == 0, np.inf, 2 * np.pi / np.where(a == 0, 1.0, a))
        low_w, high_w = mp / c["factor1"], mp / c["factor2"]
        smooth = (mp / wavelen - c["factor1"]) / (c["factor2"] - c["factor1"])
        mid = (1 - smooth) * a / c["scale"] + smooth * a
        a = np.where(wavelen < high_w, a, np.where(wavelen > low_w, a / c["scale"], mid))
        da = da + 4.0 + 6.0 * (mp / wavelen + c["factor1"]) / (c["factor2"] - c["factor1"])
    return a, sc, np.abs(a) * da * 2.0 ** -24


def rope_plain_angle_np(base, head_dim, i, pos) -> Tuple[np.ndarray, np.ndarray]:
    """Float64 angle pos * base^(-2i/D) of the plain RoPE kernels (rope_append_kernel, the persistent kernel's rope op, the
    attention kernel's fused rope) and dA, a bound on their fp32 angle's distance from it. The kernel forms
    e = fl(fl(-2i / D) * l2b), l2b = log2(base) rounded to fp32 on the host (within 1 ulp), then exp2f(e) (2 ulp) and
    fl(pos * that). e is within 3 u |e| of the exact exponent (u = 2^-24), which moves 2^e by ln 2 * 3 u |e| relatively;
    exp2f adds 4 u, the product u: dA = |a| * u * (5 + 2.08 |e|). At i = 0 the kernel's angle is exact (e = -0, 2^e = 1),
    everywhere else dA grows like |a|: about 0.04 rad at position 131071 for the first pairs, which no fp32 RoPE avoids."""
    base = float(np.float32(base))
    i = np.asarray(i, np.float64)
    pos = np.asarray(pos, np.float64)
    e = -2.0 * i / head_dim * np.log2(base)
    a = pos * 2.0 ** e
    return a, np.abs(a) * 2.0 ** -24 * (5.0 + 3.0 * np.log(2.0) * np.abs(e))


def rope_np(qkv, head_num, kv_head_num, head_dim, positions, base=None, cfg=None, bias=None, cos_sin_cache=None,
            use_logn=False, is_bf16=False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Float64 RoPE of one token per row: qkv [B, (Hq + 2 Hkv) * D] T values (or bits), positions [B] (already resolved:
    position_ids where > 0, else the slot). The plain kernels: base given, cfg None (Base style, rotary dim = D). The
    rope_append_ex contract: cfg (RopeConfig fields), optional bias [(Hq + 2 Hkv) * D] added and rounded to T first,
    cos_sin_cache fp32 [P, dim] interleaved (cos, sin) used for pos < P, logn on q heads past max_pos.
    NeoX pairing (i, i + dim / 2) inside the first `dim` channels; the rest pass through.

    Returns (out, R, dA), each [B, Hq + 2 Hkv, D]: out the rotated q / k heads and the v heads (as stored: the input,
    with the bias rounded in); R = |logn| * ||(x_i, x_(i + dim/2))|| of each element's pair (|x| past the rotary dim), dA
    the pair's angle bound (0 from the cache: the kernel uses those fp32 values as given). rope_error_budget takes them."""
    x = _vals(qkv, is_bf16)
    B = x.shape[0]
    H = head_num + 2 * kv_head_num
    x = x.reshape(B, H, head_dim).copy()
    if bias is not None:
        x = round_t(x + _vals(bias, is_bf16).reshape(1, H, head_dim), is_bf16)
    dim = head_dim if cfg is None else int(cfg["dim"])
    rot = cfg is None or int(cfg["style"]) != 0
    half = dim // 2
    pos = np.asarray(positions, np.int64)
    i = np.arange(half)
    if cfg is None:
        a, dA = rope_plain_angle_np(base, head_dim, i[None, :], pos[:, None])
        sc = 1.0
    else:
        a, sc, dA = rope_angle_np(cfg, 2 * i[None, :], pos[:, None])
    cs, sn = sc * np.cos(a), sc * np.sin(a)
    if cos_sin_cache is not None and cfg is not None:
        cache = np.asarray(cos_sin_cache, np.float64).reshape(cos_sin_cache.shape[0], -1, 2)
        hit = pos < cache.shape[0]
        rows = cache[np.where(hit, pos, 0)]
        cs = np.where(hit[:, None], rows[..., 0], cs)
        sn = np.where(hit[:, None], rows[..., 1], sn)
        dA = np.where(hit[:, None], 0.0, dA)
    out = x.copy()
    R = np.abs(x)
    dAx = np.zeros_like(x)
    qk = slice(0, head_num + kv_head_num)
    if rot:
        x0, x1 = x[:, qk, :half], x[:, qk, half:dim]
        c, s = cs[:, None, :], sn[:, None, :]
        out[:, qk, :half] = x0 * c - x1 * s
        out[:, qk, half:dim] = x1 * c + x0 * s
        nrm = np.hypot(x0, x1) * max(abs(sc), 1.0)
        R[:, qk, :half] = nrm
        R[:, qk, half:dim] = nrm
        dAx[:, qk, :half] = dA[:, None, :]
        dAx[:, qk, half:dim] = dA[:, None, :]
    if use_logn and cfg is not None:
        mp = int(cfg["max_pos"])
        L = np.where(pos > mp, np.log(pos + 1.0) / np.log(float(mp)), 1.0)[:, None, None]
        out[:, :head_num] *= L
        R[:, :head_num] *= L
    return out, R, dAx


def rope_error_budget(ref, R, dA, is_bf16: bool) -> np.ndarray:
    """Per-element bound on |y - ref| for a RoPE kernel in T against rope_np's (ref, R, dA): ulp_T(ref) + R * (dA + 16 u),
    u = 2^-24. Why: an angle off by dA rotates the pair by dA, moving each output by at most ||(x0, x1)|| dA. sincosf is
    within 2 ulp (<= 4 u absolute on cos and sin, so up to 4 sqrt(2) u ||x|| on an output), the rotation's product and
    fma round once each (2 u ||x||), Yarn's mscale product and logn's factor (two logf of 1 ulp, a division, a product:
    <= 8 u) the rest. The one final rounding to T is half an ulp_T. A position off by one moves the angle of pair 0 by
    one radian, which no budget of this form allows; a bias not rounded to T first moves an output by a fraction of an ulp_T,
    which the rounded fractions see (rope_fraction_mask)."""
    return ulp(ref, is_bf16) + np.asarray(R, np.float64) * (np.asarray(dA, np.float64) + 16 * 2.0 ** -24)


def rope_fraction_mask(ref, R, dA, is_bf16: bool) -> np.ndarray:
    """The outputs where the fp32 part of rope_error_budget is below an eighth of ulp_T(ref): there a correct kernel rounds
    almost every output correctly, so gemm_rounded_fractions against ROPE_MIN_* is a sharp check."""
    return np.asarray(R) * (np.asarray(dA) + 16 * 2.0 ** -24) <= ulp(ref, is_bf16) / 8


# ----------------------------------------------------------------------------------------------
# Weight-only quantisation
# ----------------------------------------------------------------------------------------------
def unpack_groupwise_int4(qweight, qzeros, scales_f16, group: int, is_gptq: bool):
    """device_impl.py:242-300 (4-bit). Returns (q_packed uint8 [K,N/2], zeros_x_scales f16 [K/g,N], scales f16)."""
    qweight = np.ascontiguousarray(qweight, dtype=np.int32)
    qzeros = np.ascontiguousarray(qzeros, dtype=np.int32)
    scales = np.ascontiguousarray(scales_f16, dtype=np.float16)
    if is_gptq:
        K, N = qweight.shape[0] * 8, qweight.shape[1]
    else:
        K, N = qweight.shape[0], qweight.shape[1] * 8
    qp = np.zeros((K, N // 2), np.uint8)
    zs = np.zeros((K // group, N), np.float16)
    lib().oracle_unpack_groupwise_int4(_p(qweight), _p(qzeros), _p(scales.view(np.uint16)), K, N, group,
                                       int(is_gptq), _p(qp), _p(zs.view(np.uint16)))
    return qp, zs, scales


def unpack_groupwise_int8(qweight, qzeros, scales_f16, group: int, is_gptq: bool):
    """device_impl.py:242-300 with weight_bits == 8 (is_int8: zero shift 128, one byte per weight, :147-149,256-258).
    GPTQ qweight int32 [K/4, N] (4 bytes along K, low byte first), AWQ qweight int32 [K, N/4] (bytes along N, then the
    reference applies reverse_awq_order over runs of 8 columns, :163-171,267), qzeros int32 [K/g, N/4].
    Returns (q_s int8 [K,N], zeros_x_scales f16 [K/g,N], scales f16)."""
    qweight = np.ascontiguousarray(qweight, dtype=np.int32)
    qzeros = np.ascontiguousarray(qzeros, dtype=np.int32)
    scales = np.ascontiguousarray(scales_f16, dtype=np.float16)

    def awq_order(t):                       # out[..., 8g + 2j + i] = in[..., 8g + 4i + j]
        return t.reshape(-1, 2, 4).transpose(0, 2, 1).reshape(t.shape)
    if is_gptq:
        u = np.ascontiguousarray(qweight.T).view(np.uint8).T.astype(np.int16)      # [K, N]
    else:
        u = awq_order(qweight.view(np.uint8).astype(np.int16))
    q = (u - 128).astype(np.int8)
    z = qzeros.view(np.uint8).astype(np.int16)
    if not is_gptq:
        z = awq_order(z)
    zf = (-z + 128 - (1 if is_gptq else 0)).astype(np.float16)                      # |.| <= 128: exact in fp16
    zs = (zf.astype(np.float32) * scales.astype(np.float32)).astype(np.float16)     # one rounding, as torch's half multiply
    return np.ascontiguousarray(q), zs, scales


def quantize_int8_per_col(w: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """device_impl.py:183-202 int8 branch. w [K,N] float -> (q int8 [K,N], scale fp32 [N])."""
    w = np.ascontiguousarray(w, dtype=np.float32)
    K, N = w.shape
    q = np.empty((K, N), np.int8)
    s = np.empty(N, np.float32)
    lib().oracle_quantize_int8_per_col(_p(w), K, N, _p(q), _p(s))
    return q, s


def unpack_int4_signed(q_packed: np.ndarray) -> np.ndarray:
    """[K,N/2] uint8 -> q_s int8 [K,N] in [-8,7] (low nibble = even column, device_impl.py:204-209)."""
    lo = (q_packed & 0xF).astype(np.int8)
    hi = (q_packed >> 4).astype(np.int8)
    lo = np.where(lo >= 8, lo - 16, lo)
    hi = np.where(hi >= 8, hi - 16, hi)
    out = np.empty((q_packed.shape[0], q_packed.shape[1] * 2), np.int8)
    out[:, 0::2] = lo
    out[:, 1::2] = hi
    return out


def dequant_np(fmt: str, weight, scales=None, zeros_x_scales=None, group: int = 128, is_bf16=False) -> np.ndarray:
    """W' [K,N] float32 per SURVEY section 8 a9/a10 (rounded to the activation type)."""
    def rnd(x):
        return from_bits(to_bits(x, is_bf16), is_bf16)
    if fmt == "f16":
        return np.asarray(weight, np.float32)
    if fmt == "int8":
        return rnd(weight.astype(np.float32) * np.asarray(scales, np.float32)[None, :])
    if fmt == "int4":
        qs = unpack_int4_signed(weight).astype(np.float32)
        s = np.repeat(np.asarray(scales, np.float32), group, axis=0)
        z = np.repeat(np.asarray(zeros_x_scales, np.float32), group, axis=0)
        return rnd(qs * s + z)
    if fmt == "int8g":
        s = np.repeat(np.asarray(scales, np.float32), group, axis=0)
        z = np.repeat(np.asarray(zeros_x_scales, np.float32), group, axis=0)
        return rnd((np.asarray(weight).astype(np.float64) * s + z).astype(np.float32))   # fma: one rounding to fp32, then to the element type
    raise ValueError(fmt)


_FMT = {"f16": 0, "int8": 1, "int4": 2, "int8g": 3}


def dequant_gemm(x_bits, fmt: str, weight, scales=None, zeros_x_scales=None, group: int = 128, bias=None,
                 is_bf16=False, fast=False) -> np.ndarray:
    """Y = X . W' (+bias). x_bits [B,K] uint16; weight per fmt (f16: uint16 bits [K,N]; int8: int8 [K,N];
    int4: uint8 [K,N/2]; int8g: int8 [K,N]); scales / zeros as uint16 bits (int8: [N]; int4 / int8g: [K/g,N]).
    Returns bits [B,N]."""
    x_bits = np.ascontiguousarray(x_bits, dtype=np.uint16)
    B, K = x_bits.shape
    weight = np.ascontiguousarray(weight)
    N = weight.shape[1] * (2 if fmt == "int4" else 1)
    y = np.empty((B, N), np.uint16)
    sc = to_bits(np.asarray(scales), is_bf16) if scales is not None else None
    zs = to_bits(np.asarray(zeros_x_scales), is_bf16) if zeros_x_scales is not None else None
    bs = to_bits(np.asarray(bias), is_bf16) if bias is not None else None
    if fast:
        assert bias is None
        lib().oracle_dequant_gemm_fast(_p(x_bits), int(is_bf16), B, K, N, _FMT[fmt], _p(weight),
                                       _p(sc) if sc is not None else None, _p(zs) if zs is not None else None,
                                       int(group), _p(y))
    else:
        lib().oracle_dequant_gemm(_p(x_bits), int(is_bf16), B, K, N, _FMT[fmt], _p(weight),
                                  _p(sc) if sc is not None else None, _p(zs) if zs is not None else None,
                                  int(group), _p(bs) if bs is not None else None, _p(y))
    return y


# ----------------------------------------------------------------------------------------------
# Glue ops
# ----------------------------------------------------------------------------------------------
def add_rmsnorm(x_bits, residual_bits, gamma_bits, eps, is_bf16=False):
    x_bits = np.ascontiguousarray(x_bits, np.uint16)
    rows, hidden = x_bits.shape
    y = np.empty_like(x_bits)
    res = np.ascontiguousarray(residual_bits, np.uint16).copy() if residual_bits is not None else None
    lib().oracle_add_rmsnorm(_p(x_bits), _p(res) if res is not None else None,
                             _p(np.ascontiguousarray(gamma_bits, np.uint16)), _p(y), int(is_bf16), rows, hidden,
                             ctypes.c_float(eps), int(res is not None))
    return y, res


def silu_and_mul(gate_up_bits, is_bf16=False):
    g = np.ascontiguousarray(gate_up_bits, np.uint16)
    rows, two_inter = g.shape
    y = np.empty((rows, two_inter // 2), np.uint16)
    lib().oracle_silu_and_mul(_p(g), _p(y), int(is_bf16), rows, two_inter // 2)
    return y


def rope_append(qkv_bits, kv_pool_bits, page_list, sequence_lengths, head_num, kv_head_num, head_dim,
                tokens_per_block, rope_base, is_bf16=False):
    """Returns (q_out bits [B,Hq*D], updated kv_pool bits copy)."""
    qkv = np.ascontiguousarray(qkv_bits, np.uint16)
    pool = np.ascontiguousarray(kv_pool_bits, np.uint16).copy()
    page_list = np.ascontiguousarray(page_list, np.int32)
    seq = np.ascontiguousarray(sequence_lengths, np.int32)
    B = qkv.shape[0]
    q_out = np.empty((B, head_num * head_dim), np.uint16)
    lib().oracle_rope_append(_p(qkv), _p(q_out), _p(pool), _p(page_list), _p(seq), int(is_bf16), B, head_num,
                             kv_head_num, head_dim, page_list.shape[-1], tokens_per_block, ctypes.c_float(rope_base))
    return q_out, pool


def argmax(logits: np.ndarray) -> np.ndarray:
    logits = np.ascontiguousarray(logits, np.float32)
    out = np.empty(logits.shape[0], np.int32)
    lib().oracle_argmax(_p(logits), logits.shape[0], logits.shape[1], _p(out))
    return out


def sample(logits, top_k, top_p, uniform, temperature=None, history=None, hist_len=None, repetition=None, presence=None,
           frequency=None, process=None):
    """sampleGreedy's path on fp32 logits [B, V]. Returns (tokens, token_prob, probs after softmax, renormalised kept probs)."""
    lg = np.ascontiguousarray(logits, np.float32).copy()
    B, V = lg.shape
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    hist = None if history is None else np.ascontiguousarray(history, np.int32)
    hl = None if hist_len is None else np.ascontiguousarray(hist_len, np.int32)
    tk, tp, u = np.ascontiguousarray(top_k, np.int32), f32(top_p), f32(uniform)
    t, rp, pp, fp = f32(temperature), f32(repetition), f32(presence), f32(frequency)
    pr = None if process is None else np.ascontiguousarray(process, np.uint8)
    tok = np.empty(B, np.int32)
    tprob = np.empty(B, np.float32)
    probs = np.empty((B, V), np.float32)
    P = lambda a: None if a is None else _p(a)
    lib().oracle_sample(_p(lg), B, V, P(hist), P(hl), hist.shape[1] if hist is not None else 0, P(t), P(rp), P(pp), P(fp), _p(tk),
                        _p(tp), _p(u), P(pr), _p(tok), _p(tprob), _p(probs))
    return tok, tprob, lg, probs


class RopeConfig(ctypes.Structure):
    _fields_ = [("style", ctypes.c_int), ("dim", ctypes.c_int), ("base", ctypes.c_float), ("scale", ctypes.c_float),
                ("factor1", ctypes.c_float), ("factor2", ctypes.c_float), ("max_pos", ctypes.c_int),
                ("extrapolation_factor", ctypes.c_float), ("mscale", ctypes.c_float)]


def rope_append_ex(qkv_bits, kv_pool_bits, page_list, sequence_lengths, head_num, kv_head_num, head_dim, tokens_per_block, cfg,
                   bias_bits=None, position_ids=None, cos_sin_cache=None, use_logn=False, is_bf16=False):
    """The full decode rope contract (b200_rope_append_ex). cfg: dict of RopeConfig fields. Returns (q_out bits, pool copy)."""
    qkv = np.ascontiguousarray(qkv_bits, np.uint16)
    pool = np.ascontiguousarray(kv_pool_bits, np.uint16).copy()
    page_list = np.ascontiguousarray(page_list, np.int32)
    seq = np.ascontiguousarray(sequence_lengths, np.int32)
    B = qkv.shape[0]
    q_out = np.empty((B, head_num * head_dim), np.uint16)
    rc = RopeConfig(**cfg)
    bias = None if bias_bits is None else np.ascontiguousarray(bias_bits, np.uint16)
    pid = None if position_ids is None else np.ascontiguousarray(position_ids, np.int32)
    cache = None if cos_sin_cache is None else np.ascontiguousarray(cos_sin_cache, np.float32)
    P = lambda a: None if a is None else _p(a)
    lib().oracle_rope_append_ex(_p(qkv), P(bias), _p(q_out), _p(pool), _p(page_list), _p(seq), P(pid), P(cache),
                                cache.shape[0] if cache is not None else 0, ctypes.byref(rc), int(use_logn), int(is_bf16), B, head_num,
                                kv_head_num, head_dim, page_list.shape[-1], tokens_per_block)
    return q_out, pool


def rope_cache_base(dim, theta, scale, max_pos):
    """genBaseCache (cpp/model_utils/RopeCache.cc:16-44), interleave = true: fp32 [positions, dim] = (cos, sin) pairs."""
    inv_freq = (1.0 / np.power(np.float32(theta), np.arange(0, dim, 2, dtype=np.float32) / np.float32(dim))).astype(np.float32)
    t = (np.arange(int(max_pos * scale), dtype=np.float32) / np.float32(scale)).astype(np.float32)
    freqs = np.outer(t, inv_freq).astype(np.float32)
    return np.stack([np.cos(freqs), np.sin(freqs)], axis=-1).reshape(freqs.shape[0], -1).astype(np.float32)


def rope_cache_yarn(dim, theta, scale, max_pos, beta_slow, beta_fast, extrapolation_factor, mscale):
    """genYarnCache (RopeCache.cc:46-85), interleave = true."""
    pos_freqs = np.power(np.float32(theta), np.arange(0, dim, 2, dtype=np.float32) / np.float32(dim)).astype(np.float32)
    inv_e, inv_i = (1.0 / pos_freqs).astype(np.float32), (1.0 / (np.float32(scale) * pos_freqs)).astype(np.float32)

    def corr(nrot):
        return np.float32(dim * np.log(np.float32(max_pos / (nrot * 2.0 * np.pi)))) / (2.0 * np.log(np.float32(theta)))
    low = float(max(0, int(np.floor(corr(beta_slow)))))
    high = float(min(dim - 1, int(np.ceil(corr(beta_fast)))))
    if abs(low - high) < 1e-6:
        high += 0.001
    ramp = np.clip((np.arange(dim // 2, dtype=np.float32) - low) / (high - low), 0, 1).astype(np.float32)
    mask = ((1.0 - ramp) * extrapolation_factor).astype(np.float32)
    inv_freq = (inv_i * (1.0 - mask) + inv_e * mask).astype(np.float32)
    t = np.arange(int(max_pos * scale), dtype=np.float32)
    freqs = np.outer(t, inv_freq).astype(np.float32)
    return (np.stack([np.cos(freqs), np.sin(freqs)], axis=-1).reshape(freqs.shape[0], -1) * np.float32(mscale)).astype(np.float32)


def qk_rmsnorm(qkv_bits, q_gamma_bits, k_gamma_bits, head_num, kv_head_num, head_dim, eps, q_bias_bits=None, k_bias_bits=None,
               is_bf16=False):
    x = np.ascontiguousarray(qkv_bits, np.uint16).copy()
    c = lambda a: None if a is None else _p(np.ascontiguousarray(a, np.uint16))
    qg, kg = np.ascontiguousarray(q_gamma_bits, np.uint16), np.ascontiguousarray(k_gamma_bits, np.uint16)
    qb = None if q_bias_bits is None else np.ascontiguousarray(q_bias_bits, np.uint16)
    kb = None if k_bias_bits is None else np.ascontiguousarray(k_bias_bits, np.uint16)
    lib().oracle_qk_rmsnorm(_p(x), _p(qg), _p(kg), None if qb is None else _p(qb), None if kb is None else _p(kb), int(is_bf16),
                            x.shape[0], head_num, kv_head_num, head_dim, ctypes.c_float(eps))
    return x
