"""Numpy references of speculative verification, used by the CPU and GPU tests:

- verify_np: spec_verify_kernel's walk over a token tree and its three accept rules (b200_spec_verify_tree and
  b200_spec_verify_tree_draft), each rule in float32 operation for operation as the kernel takes it, so its decisions are the
  kernel's bit for bit; chain_verify_np: b200_spec_verify, the same walk on the chain parent(c) = c - 1;
- block_sum_f32: the kernel's order of the sum Z of a draft-rows residual;
- ancestors, compact_np, random_tree: the visible sets of b200_paged_decode_attn_tree, b200_kv_compact_path, test trees;
- verify_measure / exact_emitted / extend / target_joint: the float64 measure of the emitted tokens under the rules, with the
  accept tests integrated exactly, for the unbiasedness theorems."""
import itertools
from collections import defaultdict

import numpy as np

THREADS = 1024
F32 = np.float32


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


def block_sum_f32(r: np.ndarray) -> np.float32:
    """sum(r) in the kernel's order (spec_residual_pass + block_reduce_sum): thread k adds, in index order, the elements of the
    4-element groups k, k + 1024, ...; each warp folds its 32 lanes by xor shuffles 16, 8, 4, 2, 1 and lane 0's value stands
    for the warp; the 32 warp sums are added in warp order from 0."""
    r = np.asarray(r, F32)
    G = -(-r.size // 4)
    K = -(-G // THREADS)
    pad = np.zeros(K * THREADS * 4, F32)
    pad[:r.size] = r
    a = pad.reshape(K, THREADS, 4)
    part = np.zeros(THREADS, F32)
    for k in range(K):
        for j in range(4):
            part = part + a[k, :, j]
    lanes = part.reshape(THREADS // 32, 32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, idx ^ o]
    total = F32(0)
    for w in lanes[:, 0]:
        total = F32(total + w)
    return total


# ---------------------------------------------------------------------------------------------------- the verifier
def _deterministic(t, toks, kids, u):
    """Drafts as fixed tokens: child c with token x is accepted iff fl(u[c-1] * fl(1 - S)) < r(x), r the row t with the tokens of
    the siblings rejected before c zeroed and S the fp32 running sum of r over those rejections. Returns the accepted child, or
    None and the residual max(0, t - 1) on the rejected tokens."""
    S, rejected = F32(0), []
    for c in kids:
        x = int(toks[c])
        q = t[x] if 0 <= x < t.size and x not in rejected else F32(0)
        if F32(u[c - 1]) * F32(F32(1) - S) < q:
            return c, None
        S = F32(S + q)
        rejected.append(x)
    sub = np.zeros_like(t)
    sub[[x for x in rejected if 0 <= x < t.size]] = 1
    return None, np.maximum(F32(0), t - sub)


def _draft_rows(t, rows, toks, kids, u):
    """Drafts with their rows (SpecInfer's recursive rejection): with R = t and Z = 1, child c with token x and row p = rows[c] is
    accepted iff fl(fl(u[c-1] * p(x)) * Z) < R(x); on a rejection R = max(0, fl(R - fl(Z * p))) and Z = block_sum_f32(R).
    Returns the accepted child, or None and R."""
    R, Z = t, F32(1)
    for c in kids:
        x = int(toks[c])
        inside = 0 <= x < t.size
        if F32(F32(F32(u[c - 1]) * (rows[c, x] if inside else F32(0))) * Z) < (R[x] if inside else F32(0)):
            return c, None
        R = np.fmax(F32(0), R - Z * rows[c])
        Z = block_sum_f32(R)
    return None, R


def verify_np(parents, node_tokens, *, target_ids=None, target_probs=None, draft_probs=None, uniform=None):
    """spec_verify_kernel on a token tree in numpy. parents, node_tokens [B, n] (node 0 the root, whose token is not read). The
    rule is picked as the C ABI picks it: target_ids [B, n] greedy; target_probs [B, n, V] with uniform [B, n] deterministic
    drafts, and with draft_probs [B, n, V] (node c's row at c, row 0 unread) draft rows.
    From the root the walk tests the current node's children (parents[c] == cur, c > cur) in index order, moves to the first one
    accepted and stops at a leaf or when every child is rejected. Greedy accepts the first child whose token is
    target_ids[cur] and emits target_ids[cur]; the sampling rules (_deterministic, _draft_rows) draw the emitted token from the
    residual their rejections left (from t when that has no mass, and at a leaf) by _draw_np with uniform[n - 1].
    Returns (out_tokens int32 [B, n], accepted int32 [B], accepted_path int32 [B, n], draw_mass): draw_mass[b] the mass
    sequence b's draw used, None in greedy."""
    par = np.asarray(parents, np.int64)
    tok = np.asarray(node_tokens, np.int64)
    B, n = par.shape
    greedy = target_ids is not None
    if greedy:
        ids = np.asarray(target_ids)
    else:
        t_all = np.asarray(target_probs, F32)
        u_all = np.asarray(uniform, np.float64)
        rows = None if draft_probs is None else np.asarray(draft_probs, F32)
    out = np.full((B, n), -1, np.int32)
    acc = np.zeros(B, np.int32)
    path_out = np.full((B, n), -1, np.int32)
    draw_mass = []

    def rule(b, cur, kids):
        if greedy:
            return next((c for c in kids if tok[b, c] == ids[b, cur]), None), None
        if rows is None:
            return _deterministic(t_all[b, cur], tok[b], kids, u_all[b])
        return _draft_rows(t_all[b, cur], rows[b], tok[b], kids, u_all[b])
    for b in range(B):
        path = [0]
        while True:
            kids = _kids(par[b], path[-1])
            nxt, residual = rule(b, path[-1], kids) if kids else (None, None)
            if nxt is None:
                break
            path.append(nxt)
        cur = path[-1]
        if greedy:
            mass, x = None, int(ids[b, cur])
        else:
            t = t_all[b, cur]
            mass = residual if residual is not None and residual.astype(np.float64).sum() > 0 else np.where(t > 0, t, F32(0))
            x = _draw_np(mass, u_all[b, n - 1])
        draw_mass.append(mass)
        a = len(path) - 1
        out[b, :a] = tok[b, path[1:]]
        out[b, a] = x
        acc[b] = a
        path_out[b, :a + 1] = path
    return out, acc, path_out, draw_mass


def chain_verify_np(draft_tokens, target_probs=None, target_ids=None, draft_probs=None, uniform=None):
    """b200_spec_verify in numpy: verify_np on the chain of n + 1 nodes parent(c) = c - 1, node c's token draft_tokens[c - 1].
    draft_tokens [B, n]; target_ids [B, n + 1], or target_probs [B, n + 1, V] and uniform [B, n + 1] with draft_probs [B, n, V]
    (node c's row at c - 1) or without. Returns verify_np's (out_tokens [B, n + 1], accepted, accepted_path, draw_mass)."""
    d = np.asarray(draft_tokens, np.int64)
    B, n = d.shape
    parents = np.tile(np.arange(-1, n), (B, 1))
    tokens = np.concatenate([np.full((B, 1), -1), d], axis=1)
    if draft_probs is not None:
        dp = np.asarray(draft_probs, F32)
        draft_probs = np.concatenate([np.zeros_like(dp[:, :1]), dp], axis=1)
    return verify_np(parents, tokens, target_ids=target_ids, target_probs=target_probs, draft_probs=draft_probs, uniform=uniform)


# ---------------------------------------------------------------------------------------------------- trees
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


# ---------------------------------------------------------------------------------------------------- the exact measure
def _kids(parents, cur):
    return [c for c in range(cur + 1, len(parents)) if parents[c] == cur]


def verify_measure(parents, toks, rows, target, rule="draft", cur=0, prefix=()):
    """{emitted tokens: probability} of the verification of one drafted tree (toks[c], rows[c]: node c's token and draft row)
    from node cur, whose token path is prefix, in float64, the accept tests integrated exactly; target(path) is the target row
    after a token path. rule "draft": accept with min(1, R(x) / (Z p(x))), R = max(0, R - Z p) and Z = sum R after a
    rejection, the final draw from R / Z (t when Z is 0). rule "deterministic" (b200_spec_verify_tree's): accept with
    min(1, r(x) / (1 - S)), r the row with rejected tokens zeroed and S their mass, the final draw from r / sum r."""
    t = target(prefix)
    R, Z, reach, out = t.copy(), 1.0, 1.0, defaultdict(float)
    kids = _kids(parents, cur)
    for c in kids:
        x = toks[c]
        if rule == "draft":
            p = rows[c]
            a = (min(1.0, R[x] / (Z * p[x])) if Z * p[x] > 0 else float(R[x] > 0))
        else:
            a = min(1.0, R[x] / Z) if Z > 0 else float(R[x] > 0)
        if a > 0:
            for seq, pr in verify_measure(parents, toks, rows, target, rule, c, prefix + (x,)).items():
                out[(x,) + seq] += reach * a * pr
        reach *= 1.0 - a
        if rule == "draft":
            R = np.maximum(0.0, R - Z * rows[c])
            Z = R.sum()
        else:
            Z -= R[x]
            R[x] = 0.0
    final = R / R.sum() if kids and R.sum() > 0 else t
    for v in np.nonzero(final > 0)[0]:
        out[(int(v),)] += reach * final[v]
    return out


def _node_paths(parents, toks):
    """Each node's token path from the root (the root's is empty)."""
    paths = [()]
    for c in range(1, len(parents)):
        paths.append(paths[parents[c]] + (toks[c],))
    return paths


def exact_emitted(parents, draft, target, V, rule="draft", without_replacement=False):
    """The float64 measure of the emitted tokens (the accepted path's, then the correction or bonus token) over every draft of
    the tree and every uniform. draft(prefix) is the drafter's row for a child of the node with token path prefix; with
    without_replacement a node's row is that row with the tokens of its earlier siblings removed and renormalised (the row the
    verifier is given). rule "deterministic" verifies the same drafts by b200_spec_verify_tree's rule. Returns {tokens: p}."""
    parents = [int(x) for x in parents]
    n = len(parents)
    out = defaultdict(float)
    for toks in itertools.product(range(V), repeat=n - 1):
        toks = (-1,) + toks
        paths = _node_paths(parents, toks)
        rows, w = [None] * n, 1.0
        for c in range(1, n):
            row = draft(paths[parents[c]]).copy()
            if without_replacement:
                for s in range(1, c):
                    if parents[s] == parents[c]:
                        row[toks[s]] = 0.0
                row = row / row.sum() if row.sum() > 0 else row
            rows[c] = row
            w *= row[toks[c]]
            if w == 0.0:
                break
        if w == 0.0:
            continue
        for seq, pr in verify_measure(parents, toks, rows, target, rule).items():
            out[seq] += w * pr
    return dict(out)


def extend(measure, target, L):
    """The measure of the emitted tokens continued by the target to L tokens: {L tokens: p}."""
    out = defaultdict(float)
    stack = list(measure.items())
    while stack:
        seq, p = stack.pop()
        if len(seq) >= L:
            out[seq[:L]] += p
            continue
        t = target(seq)
        for v in np.nonzero(t > 0)[0]:
            stack.append((seq + (int(v),), p * t[v]))
    return dict(out)


def target_joint(target, V, L):
    """The target's own measure of L tokens: prod_k target(y_<k)(y_k)."""
    return extend({(): 1.0}, target, L)
