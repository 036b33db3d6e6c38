"""Numpy restatement of constrained decoding (b200_constrain_logits, include/b200_decode_ops.h), bit for bit per logits dtype,
and of b200_sample's min-p kept set. Logits travel as their raw bits (uint16 for fp16 / bf16, uint32 for fp32) so that bf16,
which numpy lacks, and NaN payloads are exact."""
import numpy as np

BITS = {"fp16": np.uint16, "bf16": np.uint16, "fp32": np.uint32}
NEG_INF = {"fp16": 0xFC00, "bf16": 0xFF80, "fp32": 0xFF800000}


def to_f32(bits: np.ndarray, dtype: str) -> np.ndarray:
    """The fp32 value of each logit (exact: fp16 and bf16 widen without rounding)."""
    if dtype == "fp16":
        return bits.view(np.float16).astype(np.float32)
    if dtype == "bf16":
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.view(np.float32)


def round_to(x: np.ndarray, dtype: str) -> np.ndarray:
    """round_T(x) of fp32 values, to nearest even (overflow to +-inf), as bits. A NaN becomes some NaN: compare NaNs as NaNs."""
    x = np.asarray(x, np.float32)
    if dtype == "fp16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).view(np.uint16)
    if dtype == "bf16":
        u = x.view(np.uint32).astype(np.uint64)
        r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
        return np.where(np.isnan(x), np.uint16(0x7FC0), r).astype(np.uint16)
    return x.view(np.uint32)


def allowed(bitmask: np.ndarray, vocab: int) -> np.ndarray:
    """bool [rows, vocab]: token t of row r is allowed iff bit t & 31 of bitmask[r][t >> 5] is set (LSB first)."""
    t = np.arange(vocab)
    words = np.asarray(bitmask).view(np.uint32)[:, t >> 5]
    return ((words >> (t & 31).astype(np.uint32)) & 1).astype(bool)


def constrain(bits: np.ndarray, dtype: str, bitmask=None, offsets=None, ids=None, values=None):
    """The logits (bits [rows, vocab]) after b200_constrain_logits, and a bool [rows, vocab] of the biased tokens (whose value,
    when NaN, may carry any payload). Masked: -inf. Allowed with a bias entry (ids in [0, vocab)): round_T(float(x) + b) with
    one fp32 add. Everything else: the input bits."""
    rows, V = bits.shape
    out = bits.copy()
    ok = np.ones((rows, V), bool) if bitmask is None else allowed(bitmask, V)
    biased = np.zeros((rows, V), bool)
    if offsets is not None:
        offsets = np.asarray(offsets, np.int64)
        r = np.repeat(np.arange(rows), np.diff(offsets))
        t = np.asarray(ids, np.int64)[offsets[0]:offsets[-1]]
        b = np.asarray(values, np.float32)[offsets[0]:offsets[-1]]
        keep = (t >= 0) & (t < V)
        r, t, b = r[keep], t[keep], b[keep]
        keep = ok[r, t]
        r, t, b = r[keep], t[keep], b[keep]
        with np.errstate(invalid="ignore", over="ignore"):                  # inf + -inf, and fp32 overflow, are the contract
            out[r, t] = round_to(to_f32(bits[r, t], dtype) + b, dtype)
        biased[r, t] = True
    out[~ok] = NEG_INF[dtype]
    return out, biased


def min_p_kept(p: np.ndarray, base_kept: np.ndarray, min_p) -> np.ndarray:
    """b200_sample's kept set with min-p: the top-k / top-p kept set (base_kept) intersected with p >= fl32(min_p * max p),
    per row of the kernel's own fp32 probabilities p, min_p clamped to [0, 1]."""
    mp = np.clip(np.asarray(min_p, np.float32), np.float32(0), np.float32(1))
    thr = (mp * p.max(axis=-1)).astype(np.float32)
    return base_kept & (p >= thr[:, None])
