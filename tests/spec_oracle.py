"""Numpy reference of b200_spec_verify (speculative-token verification), used by the CPU and GPU tests."""
import numpy as np


def _draw_np(mass: np.ndarray, u: float) -> int:
    """Inverse CDF in index order over non-negative masses, in float64: the first index whose running sum exceeds u * total
    (the last index with mass when rounding leaves none); -1 when nothing has mass."""
    m = mass.astype(np.float64)
    total = m.sum()
    if not total > 0.0:
        return -1
    idx = np.nonzero(m > 0.0)[0]
    c = np.cumsum(m[idx])
    k = int(np.searchsorted(c, float(u) * total, side="right"))
    return int(idx[min(k, idx.size - 1)])


def spec_verify_np(draft_tokens, target_probs=None, target_ids=None, draft_probs=None, uniform=None):
    """b200_spec_verify in numpy. draft_tokens [B, n]. Greedy (target_probs None): target_ids [B, n+1]. Sampling: target_probs
    [B, n+1, V], draft_probs [B, n, V] or None (one-hot drafts), uniform [B, n+1]. The accept test uniform[i] * p < q is taken in
    float32 as the kernel takes it; the residual max(0, q - p) is formed in float32 and drawn in float64 with uniform[n].
    Returns (out_tokens int32 [B, n+1], accepted int32 [B])."""
    d = np.asarray(draft_tokens, np.int64)
    B, n = d.shape
    out = np.full((B, n + 1), -1, np.int32)
    acc = np.zeros(B, np.int32)
    for b in range(B):
        a = 0
        if target_probs is None:
            ids = np.asarray(target_ids)[b]
            while a < n and d[b, a] == ids[a]:
                a += 1
            tok = int(ids[a])
        else:
            t = np.asarray(target_probs, np.float32)[b]
            u = np.asarray(uniform, np.float64)[b]
            V = t.shape[-1]
            dp = None if draft_probs is None else np.asarray(draft_probs, np.float32)[b]
            while a < n:
                x = d[b, a]
                inside = 0 <= x < V
                q = t[a, x] if inside else np.float32(0)
                p = (dp[a, x] if inside else np.float32(0)) if dp is not None else np.float32(1)
                if not np.float32(u[a]) * np.float32(p) < q:      # float32, as the kernel compares
                    break
                a += 1
            if a < n:
                x = d[b, a]
                draft = dp[a] if dp is not None else (np.arange(V) == x).astype(np.float32)
                r = np.maximum(np.float32(0), t[a] - draft)
                tok = _draw_np(r, u[n]) if r.astype(np.float64).sum() > 0 else _draw_np(np.where(t[a] > 0, t[a], 0), u[n])
            else:
                tok = _draw_np(np.where(t[n] > 0, t[n], 0), u[n])
        out[b, :a] = d[b, :a]
        out[b, a] = tok
        acc[b] = a
    return out, acc
