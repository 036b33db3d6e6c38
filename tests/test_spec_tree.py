"""CPU tests of speculative token-tree verification: the argument checks of b200_paged_decode_attn_tree, b200_spec_verify_tree
and b200_kv_compact_path (rejected on the host before any CUDA call), and the numpy references of tests/tree_oracle.py, which
on a chain must be the chain verifier spec_verify_np."""
import ctypes

import numpy as np
import pytest

from rtp_llm_b200 import _lib
from tests.spec_oracle import spec_verify_np
from tests.tree_oracle import ancestors, compact_np, random_tree, tree_verify_np


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.fixture(scope="module")
def hostbuf():
    buf = (ctypes.c_uint8 * (1 << 16))()
    return buf, ctypes.cast(buf, ctypes.c_void_p)


def _attn_tree(lib, p, Hq, Hkv, q_len, parents, D=128, q=None):
    q = p if q is None else q
    return lib.b200_paged_decode_attn_tree(q, 0, p, Hq, Hkv, D, 2, q_len, 4, 256, 64, p, p, p, parents, 1.0, p, 4096, None)


def test_tree_attention_argument_checks(lib, hostbuf):
    _, p = hostbuf
    assert _attn_tree(lib, p, 8, 1, 4, None) == -1 and b"tree_parents" in lib.b200_last_error()
    assert _attn_tree(lib, p, 8, 1, 0, p) == -1 and b"q_len" in lib.b200_last_error()
    assert _attn_tree(lib, p, 8, 1, 65, p) == -1 and b"q_len" in lib.b200_last_error()
    for Hq, Hkv, q_len in [(64, 1, 2), (13, 1, 5)]:                        # 128 and 65 query rows
        assert _attn_tree(lib, p, Hq, Hkv, q_len, p) == -1 and b"64" in lib.b200_last_error()
    assert _attn_tree(lib, p, 8, 1, 4, p, D=96) == -1 and b"head_dim" in lib.b200_last_error()
    assert lib.b200_paged_decode_attn_tree(None, 0, None, 8, 1, 128, 0, 4, 4, 256, 64, None, None, None, None, 1.0, None, 0,
                                           None) == 0                   # empty batch: no work


def test_spec_verify_tree_argument_checks(lib, hostbuf):
    _, p = hostbuf
    f = lib.b200_spec_verify_tree
    assert f(None, p, p, p, None, 2, 0, 100, p, p, p, None) == -1 and b"n 0" in lib.b200_last_error()
    assert f(None, p, p, p, None, 2, 65, 100, p, p, p, None) == -1 and b"1..64" in lib.b200_last_error()
    assert f(None, p, p, p, None, 2, 4, 0, p, p, p, None) == -1 and b"vocab" in lib.b200_last_error()
    assert f(None, p, p, p, None, 70000, 4, 100, p, p, p, None) == -1 and b"batch" in lib.b200_last_error()
    for i in range(3):                                                      # tree_parents, node_tokens, then each output
        args = [p, p, p]
        args[i] = None
        assert f(None, p, args[0], args[1], None, 2, 4, 100, args[2], p, p, None) == -1 and b"null" in lib.b200_last_error()
    assert f(None, p, p, p, None, 2, 4, 100, p, None, p, None) == -1 and b"null" in lib.b200_last_error()
    assert f(None, p, p, p, None, 2, 4, 100, p, p, None, None) == -1 and b"null" in lib.b200_last_error()
    assert f(None, None, p, p, None, 2, 4, 100, p, p, p, None) == -1 and b"target" in lib.b200_last_error()
    assert f(p, None, p, p, None, 2, 4, 100, p, p, p, None) == -1 and b"uniform" in lib.b200_last_error()
    assert f(None, None, None, None, None, 0, 4, 100, None, None, None, None) == 0      # empty batch: no work


def test_kv_compact_path_argument_checks(lib, hostbuf):
    _, p = hostbuf
    pools1 = (ctypes.c_void_p * 2)(p.value, p.value)

    def f(pools=pools1, layers=2, hkv=8, D=128, T=16, pl=p, M=4, seq=p, path=p, acc=p, B=2, n=4):
        return lib.b200_kv_compact_path(pools, layers, hkv, D, T, pl, M, seq, path, acc, B, n, None)
    assert f(layers=0) == -1 and b"layers" in lib.b200_last_error()
    assert f(layers=129) == -1 and b"1..128" in lib.b200_last_error()
    assert f(hkv=0) == -1 and b"kv_head_num" in lib.b200_last_error()
    assert f(D=96) == -1 and b"head_dim" in lib.b200_last_error()
    assert f(T=0) == -1 and b"page_size" in lib.b200_last_error()
    assert f(n=0) == -1 and b"n 0" in lib.b200_last_error()
    assert f(n=65) == -1 and b"1..64" in lib.b200_last_error()
    assert f(B=-1) == -1 and b"batch" in lib.b200_last_error()
    for kw in ("pl", "seq", "path", "acc", "pools"):
        assert f(**{kw: None}) == -1 and b"null" in lib.b200_last_error(), kw
    assert f(pools=(ctypes.c_void_p * 2)(p.value, None)) == -1 and b"layer 1" in lib.b200_last_error()
    assert f(pools=(ctypes.c_void_p * 2)(p.value, p.value + 2)) == -1 and b"aligned" in lib.b200_last_error()
    assert f(B=0, pools=None, pl=None) == 0                                 # empty batch: no work


# ---------------------------------------------------------------------------------------------------- the oracles
def test_ancestor_walk():
    assert ancestors([-1, 0, 1, 2]) == [[0], [0, 1], [0, 1, 2], [0, 1, 2, 3]]
    assert ancestors([-1, 0, 0, 1, 1, 2]) == [[0], [0, 1], [0, 2], [0, 1, 3], [0, 1, 4], [0, 2, 5]]
    # a parent outside [0, i) ends the walk: node 2's parent is itself, node 3's is later, node 4 sits under node 3
    assert ancestors([7, 0, 2, 5, 3]) == [[0], [0, 1], [2], [3], [3, 4]]


@pytest.mark.parametrize("seed", range(4))
def test_tree_oracle_is_the_chain_oracle_on_chains(seed):
    rng = np.random.default_rng(seed)
    B, n, V = 48, int(rng.integers(2, 9)), 30
    par = np.tile(random_tree(rng, n, "chain"), (B, 1))
    ids = rng.integers(0, V, (B, n))
    toks = np.where(rng.random((B, n)) < 0.7, np.roll(ids, 1, axis=1), rng.integers(0, V, (B, n)))
    toks[:, 0] = -5                                                          # the root's entry is never read
    g_tree = tree_verify_np(par, toks, target_ids=ids)
    g_chain = spec_verify_np(toks[:, 1:], target_ids=ids)
    np.testing.assert_array_equal(g_tree[0], g_chain[0])
    np.testing.assert_array_equal(g_tree[1], g_chain[1])
    t = rng.random((B, n, V)).astype(np.float32) ** 3
    t[:, :, rng.integers(0, V)] = 0                                          # some draft tokens without mass
    t /= t.sum(-1, keepdims=True)
    toks2 = np.concatenate([toks[:, :1], np.array([[rng.choice(V, p=t[b, i].astype(np.float64) / t[b, i].astype(np.float64).sum())
                                                     for i in range(n - 1)] for b in range(B)])], axis=1)
    u = rng.random((B, n)).astype(np.float32)
    s_tree = tree_verify_np(par, toks2, target_probs=t, uniform=u)
    s_chain = spec_verify_np(toks2[:, 1:], target_probs=t, uniform=u)
    np.testing.assert_array_equal(s_tree[0], s_chain[0])
    np.testing.assert_array_equal(s_tree[1], s_chain[1])
    for b in range(B):
        np.testing.assert_array_equal(s_tree[2][b], [i if i <= s_tree[1][b] else -1 for i in range(n)])
    assert 0 < s_tree[1].mean() < n - 1


def test_tree_oracle_greedy_takes_the_first_matching_child_and_stops_at_none():
    par = np.array([[-1, 0, 0, 2, 2, 1]])
    toks = np.array([[0, 5, 7, 9, 8, 4]])
    ids = np.array([[7, 0, 8, 0, 3, 0]])                                     # root wants 7 (node 2), node 2 wants 8 (node 4)
    out, acc, path = tree_verify_np(par, toks, target_ids=ids)
    assert acc[0] == 2 and list(path[0]) == [0, 2, 4, -1, -1, -1] and list(out[0]) == [7, 8, 3, -1, -1, -1]


def test_tree_oracle_multi_round_rejection_reproduces_the_target():
    """Two deterministic siblings under the root: the first token is distributed as the root row t, whatever the drafts. The
    accept tests are integrated over a midpoint grid of (u0, u1), fine enough for these dyadic masses; the residual draw
    enters as its exact distribution."""
    t = (np.array([5, 27, 12, 20]) / 64).astype(np.float32)
    grid = (np.arange(128) + 0.5) / 128
    for d1, d2 in [(1, 3), (0, 2), (2, 2), (3, 1)]:
        par = np.array([[-1, 0, 0]])
        toks = np.array([[0, d1, d2]])
        probs = np.stack([t, t, t])[None]
        P = np.zeros(4)
        for u0 in grid:
            for u1 in grid:
                out, acc, _ = tree_verify_np(par, toks, target_probs=probs, uniform=np.array([[u0, u1, 0.5]], np.float32))
                if acc[0] == 1:
                    P[out[0, 0]] += 1
                else:                                                    # both rejected: the residual, exactly
                    r = t.astype(np.float64).copy()
                    r[[d1, d2]] = 0
                    P += r / r.sum() if r.sum() > 0 else t
        P /= len(grid) ** 2
        np.testing.assert_allclose(P, t, atol=0.01, err_msg=f"drafts {d1}, {d2}")


def test_compaction_oracle_reads_every_source_before_writing():
    slots = np.arange(10) * 10
    np.testing.assert_array_equal(compact_np(slots, 4, [0, 2, 3], 2), [0, 10, 20, 30, 40, 60, 70, 70, 80, 90])
    np.testing.assert_array_equal(compact_np(slots, 4, [0, 1, 2], 2), slots)
    np.testing.assert_array_equal(compact_np(slots, 4, [0, 3, 5], 0), slots)


def test_decode_step_rejects_a_tree_of_one_node():
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    with pytest.raises(ValueError, match="q_len >= 2"):
        DecodeStep(TINY, 4, 40, None, q_len=1, tree=[-1])
