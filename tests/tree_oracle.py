"""Numpy references of speculative token-tree verification: the ancestor sets of b200_paged_decode_attn_tree, the verifier
b200_spec_verify_tree and the path compaction b200_kv_compact_path. Used by the CPU and GPU tests."""
import numpy as np

from tests.spec_oracle import _draw_np


def ancestors(parents_row) -> list:
    """Node j's visible new tokens: j, then its parent, ... until the root or a parent outside [0, i), which ends the walk."""
    par = [int(x) for x in parents_row]
    out = []
    for j in range(len(par)):
        s, i = [j], j
        while i > 0 and 0 <= par[i] < i:
            i = par[i]
            s.append(i)
        out.append(sorted(s))
    return out


def tree_verify_np(parents, node_tokens, target_probs=None, target_ids=None, uniform=None):
    """b200_spec_verify_tree in numpy. parents, node_tokens [B, n]. Greedy: target_ids [B, n]. Sampling: target_probs [B, n, V],
    uniform [B, n]. At node cur the children c (parents[c] == cur, c > cur) are tried in index order: greedy takes the first whose
    token is target_ids[cur]; sampling accepts c iff fp32(uniform[c-1]) * fp32(1 - S) < r(x_c), r the row with the tokens of the
    siblings rejected before c zeroed and S the fp32 running sum of r over those rejections. With every child rejected the token
    is drawn from max(0, t - 1) on the rejected tokens (t when that has no mass), at a leaf from t, with uniform[n-1].
    Returns (out_tokens int32 [B, n], accepted int32 [B], accepted_path int32 [B, n])."""
    par = np.asarray(parents, np.int64)
    tok_ = np.asarray(node_tokens, np.int64)
    B, n = par.shape
    out = np.full((B, n), -1, np.int32)
    acc = np.zeros(B, np.int32)
    path_out = np.full((B, n), -1, np.int32)
    for b in range(B):
        kids = lambda cur: [c for c in range(cur + 1, n) if par[b, c] == cur]
        path = [0]
        cur = 0
        if target_probs is None:
            ids = np.asarray(target_ids)[b]
            while True:
                nxt = next((c for c in kids(cur) if tok_[b, c] == ids[cur]), None)
                if nxt is None:
                    break
                cur = nxt
                path.append(cur)
            tok = int(ids[cur])
        else:
            t_all = np.asarray(target_probs, np.float32)[b]
            u = np.asarray(uniform, np.float64)[b]
            V = t_all.shape[-1]
            while True:
                t = t_all[cur]
                S = np.float32(0)
                rejected = []
                nxt = None
                for c in kids(cur):
                    x = int(tok_[b, c])
                    inside = 0 <= x < V
                    q = t[x] if inside and x not in rejected else np.float32(0)
                    if np.float32(u[c - 1]) * np.float32(np.float32(1) - S) < q:
                        nxt = c
                        break
                    S = np.float32(S + q)
                    rejected.append(x)
                if nxt is None:
                    break
                cur = nxt
                path.append(cur)
            t = t_all[cur]
            if rejected:
                sub = np.zeros(V, np.float32)
                for x in rejected:
                    if 0 <= x < V:
                        sub[x] = 1
                r = np.maximum(np.float32(0), t - sub)
                tok = _draw_np(r, u[n - 1]) if r.astype(np.float64).sum() > 0 else _draw_np(np.where(t > 0, t, 0), u[n - 1])
            else:
                tok = _draw_np(np.where(t > 0, t, 0), u[n - 1])
        a = len(path) - 1
        out[b, :a] = tok_[b, path[1:]]
        out[b, a] = tok
        acc[b] = a
        path_out[b, :a + 1] = path
    return out, acc, path_out


def compact_np(pool_slots: np.ndarray, seq: int, path, accepted: int) -> np.ndarray:
    """b200_kv_compact_path on one sequence's slots [..., slots, ...] (slot axis 0): slot seq + d <- slot seq + path[d] for
    d = 1 .. accepted, every source read before any write (the kernel's result for an increasing path)."""
    out = pool_slots.copy()
    for d in range(1, accepted + 1):
        out[seq + d] = pool_slots[seq + path[d]]
    return out


def random_tree(rng, n: int, kind: str = "random") -> np.ndarray:
    """Parents of an n-node tree: 'chain', 'star' (every node under the root), 'binary' (node j under (j - 1) // 2) or 'random'
    (node j under a uniform earlier node)."""
    par = np.full(n, -1, np.int32)
    for j in range(1, n):
        par[j] = {"chain": j - 1, "star": 0, "binary": (j - 1) // 2}.get(kind, None) if kind != "random" else rng.integers(0, j)
    return par
