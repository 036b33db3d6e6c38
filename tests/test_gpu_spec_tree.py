"""GPU tests (H100) of speculative token-tree verification: tree-masked paged attention against a float64 oracle that gathers each
query's visible K/V into a contiguous sequence, bit equality with the q_len instance on chains and under NaN / inf in the slots a
query does not see; the tree verifier against tests/tree_oracle.py and, on chains, against b200_spec_verify bit for bit; and the
accepted-path K/V compaction, eagerly and under graph capture."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests.test_gpu_spec_verify import ROWS, V_FULL, _check_draws, _probs  # noqa: E402
from tests.tree_oracle import ancestors, compact_np, random_tree, tree_verify_np  # noqa: E402

DEV = torch.device("cuda")
TREE_ROWS = [r for r in ROWS if r[3] > 1]          # the q_len > 1 rows: D 64 / 128 / 256, fp16 / bf16, pages 16..128, RT 1 / 2 / 4
KINDS = ["chain", "star", "binary", "random", "invalid"]


def _parents(kind, B, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "invalid":     # per request: random trees with entries outside [0, j), including huge and negative ones
        par = np.stack([random_tree(rng, n, "random") for _ in range(B)])
        bad = rng.random((B, n)) < 0.4
        par[bad] = rng.choice([-7, -1, 2 ** 31 - 1, -2 ** 31, n, 64], size=int(bad.sum()))
        par[0, n - 1] = n - 1                                         # a self-parent is outside [0, j) too
        return par.astype(np.int32)
    if kind == "random":
        return np.stack([random_tree(rng, n, "random") for _ in range(B)]).astype(np.int32)
    return np.tile(random_tree(rng, n, kind), (B, 1)).astype(np.int32)


def _case(D, B, q_len, Hq, Hkv, T, lens, dtype, seed=5):
    total = [L + q_len for L in lens]
    _, pool, block_ids, _ = probe.make_attn_case(B, Hq, Hkv, T, total, dtype, seed=seed, D=D)
    q = torch.randn(B, q_len, Hq, D, generator=torch.Generator().manual_seed(9)).to(dtype)
    return q, pool, block_ids, torch.tensor(lens, dtype=torch.int32), max(total)


def _run_tree(q, pool, block_ids, seq, par, max_len, fn="tree"):
    B, q_len, Hq, D = q.shape
    Hkv = pool.shape[2]
    ws = ops.attn_workspace(B * q_len, Hq, Hkv, max_len, DEV)
    pl = ops.convert_block_table(block_ids.to(DEV))
    if fn == "tree":
        out = ops.paged_decode_attn_tree(q.to(DEV), pool.to(DEV), pl, seq.to(DEV), torch.from_numpy(par).to(DEV), max_len, ws)
    else:
        out = ops.paged_decode_attn_multi(q.to(DEV), pool.to(DEV), pl, seq.to(DEV), max_len, ws)
    torch.cuda.synchronize()
    return out, ws


def _tree_attn_np(q, pool, block_ids, seq, T, par):
    """Float64 reference with its error-size term: query j of sequence b is paged_decode_attn_np over a pseudo-sequence holding
    positions 0 .. seq[b] - 1, then the slots seq[b] + i of i in anc(j), in that order."""
    B, n, Hq, D = q.shape
    qf, pf = q.float().numpy(), pool.float().numpy()
    out = np.zeros((B, n, Hq * D))
    E = np.zeros_like(out)
    for b in range(B):
        L = int(seq[b])
        for j, anc in enumerate(ancestors(par[b])):
            pos = list(range(L)) + [L + i for i in anc]
            pg = [int(block_ids[b, p // T]) for p in pos]
            kv = pf[pg, :, :, [p % T for p in pos]]                    # [len, 2, Hkv, D]
            npg = -(-len(pos) // T)
            pseudo = np.zeros((npg * T, 2, pf.shape[2], D), np.float32)
            pseudo[:len(pos)] = kv
            pseudo = pseudo.reshape(npg, T, 2, pf.shape[2], D).transpose(0, 2, 3, 1, 4)
            o, e = orc.paged_decode_attn_np(qf[b, j][None], pseudo, np.arange(npg)[None], np.array([len(pos) - 1]), T, with_abs=True)
            out[b, j], E[b, j] = o[0], e[0]
    return out, E


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", TREE_ROWS, ids=[c[0] for c in TREE_ROWS])
def test_tree_attention_vs_float64_oracle(case, kind):
    name, D, B, q_len, Hq, Hkv, T, lens, dtype, env = case
    with probe.env_set(env):
        q, pool, block_ids, seq, max_len = _case(D, B, q_len, Hq, Hkv, T, lens, dtype)
        par = _parents(kind, B, q_len, seed=q_len)
        out, ws = _run_tree(q, pool, block_ids, seq, par, max_len)
        f64, E = _tree_attn_np(q, pool, block_ids, seq.numpy(), T, par)
        ok, info = probe.budget_info(out, f64, E, dtype == torch.bfloat16)
        assert ok, f"{name} {kind}: {info}"
        assert int(ws[: B * Hkv * 4].view(torch.int32).abs().sum().item()) == 0, "semaphores not reset"


@pytest.mark.parametrize("case", TREE_ROWS, ids=[c[0] for c in TREE_ROWS])
def test_tree_attention_on_a_chain_is_the_q_len_instance_bit_for_bit(case):
    name, D, B, q_len, Hq, Hkv, T, lens, dtype, env = case
    with probe.env_set(env):
        q, pool, block_ids, seq, max_len = _case(D, B, q_len, Hq, Hkv, T, lens, dtype, seed=11)
        par = _parents("chain", B, q_len, 0)
        got, _ = _run_tree(q, pool, block_ids, seq, par, max_len)
        exp, _ = _run_tree(q, pool, block_ids, seq, par, max_len, fn="multi")
        assert torch.equal(got.view(torch.int16), exp.view(torch.int16)), name


@pytest.mark.parametrize("case", TREE_ROWS, ids=[c[0] for c in TREE_ROWS])
def test_tree_attention_ignores_nan_and_inf_outside_a_querys_ancestors(case):
    """Star tree: node k sees the cache, the root and itself. Node 1's K/V are NaN and node 2's V +inf / K -inf: every other
    query's bits are unchanged, and nodes 1 and 2 (which see their own slot) come out NaN."""
    name, D, B, q_len, Hq, Hkv, T, lens, dtype, env = case
    if q_len < 3:
        pytest.skip("needs two non-root nodes")
    with probe.env_set(env):
        q, pool, block_ids, seq, max_len = _case(D, B, q_len, Hq, Hkv, T, lens, dtype, seed=13)
        par = _parents("star", B, q_len, 0)
        clean, _ = _run_tree(q, pool, block_ids, seq, par, max_len)
        dirty = pool.clone()
        for b in range(B):
            for k, which, val in [(1, 0, float("nan")), (1, 1, float("nan")), (2, 0, -float("inf")), (2, 1, float("inf"))]:
                p = int(seq[b]) + k                                      # (which: 0 K, 1 V)
                dirty[int(block_ids[b, p // T]), which, :, p % T] = val
        got, _ = _run_tree(q, dirty, block_ids, seq, par, max_len)
        keep = [j for j in range(q_len) if j not in (1, 2)]
        assert torch.equal(got[:, keep].view(torch.int16), clean[:, keep].view(torch.int16)), name
        assert torch.isnan(got[:, 1:3].float()).all(), name


# ---------------------------------------------------------------------------------------------------- verifier
def _T(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _random_case(seed, n, B=32):
    rng = np.random.default_rng(seed)
    par = np.stack([random_tree(rng, n, rng.choice(["random", "star", "binary"])) for _ in range(B)]).astype(np.int32)
    return rng, par


@pytest.mark.parametrize("n", [2, 3, 5, 8, 12, 16])
def test_tree_verify_greedy_vs_oracle(n):
    rng, par = _random_case(n, n)
    B = par.shape[0]
    ids = rng.integers(0, V_FULL, (B, n)).astype(np.int32)
    toks = rng.integers(0, V_FULL, (B, n)).astype(np.int32)
    for b in range(B):                    # most children repeat their parent's target id, so paths go deep and branch
        for c in range(1, n):
            if rng.random() < 0.6:
                toks[b, c] = ids[b, par[b, c]]
    toks[:, 0] = -1
    out, acc, path = ops.spec_verify_tree(_T(par), _T(toks), target_ids=_T(ids))
    eo, ea, ep = tree_verify_np(par, toks, target_ids=ids)
    np.testing.assert_array_equal(acc.cpu().numpy(), ea)
    np.testing.assert_array_equal(out.cpu().numpy(), eo)
    np.testing.assert_array_equal(path.cpu().numpy(), ep)
    assert ea.max() >= min(2, n - 1)


def _residual_masses(par, toks, t, path, acc):
    """What the draw after the walk uses: the stop node's row with its (all rejected) children's tokens removed as the chain
    removes its draft (max(0, t - 1)), or the row itself at a leaf or when that has no mass."""
    def masses(b, a):
        node = path[b, a]
        row = t[b, node]
        kids = [c for c in range(node + 1, par.shape[1]) if par[b, c] == node]
        if kids:
            sub = np.zeros_like(row)
            sub[[int(toks[b, c]) for c in kids if 0 <= toks[b, c] < row.size]] = 1
            r = np.maximum(np.float32(0), row - sub)
            if r.astype(np.float64).sum() > 0:
                return r
        return np.where(row > 0, row, 0)
    return masses


@pytest.mark.parametrize("n", [2, 3, 5, 8, 12, 16])
def test_tree_verify_sampling_vs_oracle(n):
    rng, par = _random_case(100 + n, n)
    B = par.shape[0]
    t = _probs(rng, (B, n, V_FULL), 0.25)
    toks = np.zeros((B, n), np.int32)
    for b in range(B):                    # drafts drawn from the parent's row: acceptances are frequent
        for c in range(1, n):
            row = t[b, par[b, c]].astype(np.float64)
            toks[b, c] = rng.choice(V_FULL, p=row / row.sum())
    # edge rows: duplicate siblings (row 0), a mass-free root (row 1), every child rejected with an empty residual (row 2)
    par[0] = random_tree(rng, n, "star")
    toks[0, 1:] = toks[0, 1]
    t[1, 0] = 0.0
    par[2] = random_tree(rng, n, "star")
    if n > 2:
        toks[2, 2] = (toks[2, 1] + 1) % V_FULL
    t[2, 0] = 0.0
    t[2, 0, toks[2, 1:3]] = 0.3           # mass only on (up to) two children's tokens, below what u = 0.999 accepts
    u = rng.random((B, n)).astype(np.float32)
    u[0, :] = 0.999
    u[2, :] = 0.999                       # reject every child of row 2's root
    out, acc, path = ops.spec_verify_tree(_T(par), _T(toks), target_probs=_T(t), uniform=_T(u))
    eo, ea, ep = tree_verify_np(par, toks, target_probs=t, uniform=u)
    got, acc_got, path_got = out.cpu().numpy(), acc.cpu().numpy(), path.cpu().numpy()
    np.testing.assert_array_equal(path_got, ep)
    _check_draws(got, eo, acc_got, ea, _residual_masses(par, toks, t, ep, ea), u[:, n - 1].astype(np.float64))
    assert ea[1] == 0 and eo[1, 0] == -1                 # mass-free row: every child rejected, nothing to draw
    assert ea[2] == 0 and got[2, 0] in set(toks[2, 1:3].tolist())   # empty residual: drawn from the row itself
    assert ea[0] == 0 and got[0, 0] != toks[0, 1]        # duplicate siblings: the token is rejected once for all of them


@pytest.mark.parametrize("mode", ["greedy", "sampling"])
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_tree_verify_on_a_chain_is_spec_verify_bit_for_bit(n, mode):
    rng = np.random.default_rng(7 + n)
    B = 32
    par = np.tile(random_tree(rng, n, "chain"), (B, 1)).astype(np.int32)
    if mode == "greedy":
        ids = rng.integers(0, V_FULL, (B, n)).astype(np.int32)
        drafts = np.where(rng.random((B, n - 1)) < 0.8, ids[:, :n - 1], rng.integers(0, V_FULL, (B, n - 1))).astype(np.int32)
        kw = dict(target_ids=_T(ids))
    else:
        t = _probs(rng, (B, n, V_FULL), 0.25)
        drafts = np.array([[rng.choice(V_FULL, p=t[b, i].astype(np.float64) / t[b, i].astype(np.float64).sum())
                            for i in range(n - 1)] for b in range(B)], np.int32).reshape(B, n - 1)
        kw = dict(target_probs=_T(t), uniform=_T(rng.random((B, n)).astype(np.float32)))
    toks = np.concatenate([np.full((B, 1), 77, np.int32), drafts], axis=1)
    o1, a1 = ops.spec_verify(_T(drafts), **kw)
    o2, a2, p2 = ops.spec_verify_tree(_T(par), _T(toks), **kw)
    assert torch.equal(o1, o2) and torch.equal(a1, a2)
    a = a2.cpu().numpy()
    np.testing.assert_array_equal(p2.cpu().numpy(), [[i if i <= a[b] else -1 for i in range(n)] for b in range(B)])


# ---------------------------------------------------------------------------------------------------- compaction
def _compact_case(layers, B, Hkv, D, T, n, seed, dtype=torch.float16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 3 * T, B)
    M = int(max(-(-(L + n) // T) for L in lens)) + 1
    P = B * M + 1
    caches = [torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype) for _ in range(layers)]
    blocks = (torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1)[: B * M].reshape(B, M)
    return caches, blocks, lens.astype(np.int32)


def _compact_expect(caches, blocks, lens, path, acc, T):
    """Per layer and sequence: gather the slots of the sequence (every page of its row), apply compact_np, scatter back."""
    exp = [c.clone() for c in caches]
    bl = blocks.cpu().numpy()
    for li, c in enumerate(caches):
        for b in range(bl.shape[0]):
            pos = np.arange(bl.shape[1] * T)
            pg, sl = bl[b, pos // T], pos % T
            slots = c[pg, :, :, sl].cpu()                                 # [slots, 2, Hkv, D]
            new = compact_np(slots.view(torch.int16).numpy(), int(lens[b]), list(path[b]), int(acc[b]))
            exp[li][pg, :, :, sl] = torch.from_numpy(new).view(c.dtype).to(DEV)
    return exp


PATHS = {
    "hazard [0, 2, 3]": ([0, 2, 3, -1, -1, -1], 2),
    "identity": ([0, 1, 2, 3, -1, -1], 3),
    "accepted 0": ([0, 4, 5, -1, -1, -1], 0),
    "deep": ([0, 1, 3, 4, 5, -1], 4),
}


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("D,T,dtype", [(128, 16, torch.float16), (64, 64, torch.bfloat16), (256, 32, torch.float16)])
def test_kv_compact_path_moves_the_path_and_nothing_else(D, T, dtype, graph):
    layers, B, Hkv, n = 3, 6, 2, 6
    caches, blocks, lens = _compact_case(layers, B, Hkv, D, T, n, seed=D + T, dtype=dtype)
    rng = np.random.default_rng(D)
    path = np.full((B, n), -1, np.int32)
    acc = np.zeros(B, np.int32)
    names = list(PATHS)
    for b in range(B):
        if b < len(names):
            p, a = PATHS[names[b]]
        else:                                                             # a random tree's random root-to-node path
            par = random_tree(rng, n, "random")
            node = int(rng.integers(0, n))
            p = [node]
            while p[-1] > 0:
                p.append(int(par[p[-1]]))
            p = p[::-1]
            a = len(p) - 1
            p = p + [-1] * (n - len(p))
        path[b], acc[b] = p, a
    exp = _compact_expect(caches, blocks, lens, path, acc, T)
    pl = ops.convert_block_table(blocks)
    args = (pl, _T(lens), _T(path), _T(acc))
    if graph:
        gr = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.cuda.graph(gr, stream=s):
            ops.kv_compact_path(caches, *args)
        gr.replay()
    else:
        ops.kv_compact_path(caches, *args)
    torch.cuda.synchronize()
    for li in range(layers):
        assert torch.equal(caches[li].view(torch.int16), exp[li].view(torch.int16)), f"layer {li}"
