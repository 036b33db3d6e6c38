"""References of b200_spec_verify_tree_draft (recursive rejection with draft rows on a token tree), used by the CPU and GPU tests:

- tree_draft_verify_np: the rule restated in float32, operation for operation as the kernel takes it (each product and
  difference rounded apart, Z summed in the kernel's order), so its accept decisions are the kernel's bit for bit;
- block_sum_f32: that summation order;
- exact_emitted / target_joint: the float64 measure of the emitted tokens under the rule, with the accept tests integrated
  exactly, for the unbiasedness theorem."""
import itertools
from collections import defaultdict

import numpy as np

from tests.spec_oracle import _draw_np

THREADS = 1024
F32 = np.float32


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


def tree_draft_verify_np(parents, node_tokens, target_probs, draft_probs, uniform, with_residuals=False):
    """b200_spec_verify_tree_draft in numpy. parents, node_tokens [B, n]; target_probs, draft_probs [B, n, V]; uniform [B, n].
    At node cur, R = t = target_probs[cur], Z = 1; child c (in index order) with token x and row p = draft_probs[c] is accepted
    iff fl(fl(u[c-1] * p(x)) * Z) < R(x); on a rejection R = max(0, fl(R - fl(Z * p))) and Z = block_sum_f32(R). The draw
    after the walk (R, or t when R has no mass or at a leaf) is _draw_np's float64 inverse CDF with uniform[n-1].
    Returns (out_tokens int32 [B, n], accepted int32 [B], accepted_path int32 [B, n]), and with with_residuals the mass each
    sequence's draw used."""
    par = np.asarray(parents, np.int64)
    tok_ = np.asarray(node_tokens, np.int64)
    B, n = par.shape
    out = np.full((B, n), -1, np.int32)
    acc = np.zeros(B, np.int32)
    path_out = np.full((B, n), -1, np.int32)
    masses = []
    for b in range(B):
        t_all = np.asarray(target_probs[b], F32)
        d_all = np.asarray(draft_probs[b], F32)
        u = np.asarray(uniform[b], F32)
        V = t_all.shape[-1]
        path, cur = [0], 0
        while True:
            t, R, Z, nrej, nxt = t_all[cur], None, F32(1), 0, None
            for c in range(cur + 1, n):
                if par[b, c] != cur:
                    continue
                x = int(tok_[b, c])
                inside = 0 <= x < V
                r = (R[x] if nrej else t[x]) if inside else F32(0)
                px = d_all[c, x] if inside else F32(0)
                if F32(F32(u[c - 1] * px) * Z) < r:
                    nxt = c
                    break
                R = np.fmax(F32(0), (R if nrej else t) - Z * d_all[c])
                Z = block_sum_f32(R)
                nrej += 1
            if nxt is None:
                break
            cur = nxt
            path.append(cur)
        t = t_all[cur]
        mass = R if nrej and R.astype(np.float64).sum() > 0 else np.where(t > 0, t, F32(0))
        tok = _draw_np(mass, u[n - 1])
        masses.append(mass)
        a = len(path) - 1
        out[b, :a] = tok_[b, path[1:]]
        out[b, a] = tok
        acc[b] = a
        path_out[b, :a + 1] = path
    return (out, acc, path_out, masses) if with_residuals else (out, acc, path_out)


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
