"""The peer-region model of tests/peer_oracle.py, without a GPU: its region size is the library's, every word a rank pushes
lands on a slot its owner polls, no two pushed words share a slot, everything stays inside the region, and the exact
all-reduce reference sees a change of summation order."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
from rtp_llm_b200 import _lib
from tests import peer_oracle as po

WORLDS = [2, 3, 4, 5, 8]


def test_region_bytes_match_library():
    lib = _lib.load()
    for max_msg in (16, 256, 4096, 1 << 19, (1 << 20) + 48, 1 << 20, 5 * 300 * 8192 * 2 // 5):
        assert po.Layout(max_msg).region_bytes == lib.b200_peer_ar_region_bytes(ctypes.c_size_t(max_msg)), max_msg


def _rand_bits(rng, shape, bf):
    return orc.f64_to_bits(rng.standard_normal(shape), bf)


def _check_meet(lay, world, pushes, polls):
    """pushes: {src: {dst: (off, data)}}; polls: {rank: offsets}. Every rank's polled offsets are exactly the offsets pushed
    into its region, each pushed once; all lie in the two parities, 8-byte aligned."""
    for r in range(world):
        got = np.concatenate([pushes[s][r][0] for s in range(world) if s != r])
        assert len(np.unique(got)) == len(got), f"rank {r}: two pushed words share a slot"
        assert np.array_equal(np.sort(got), np.sort(polls[r])), f"rank {r}: pushed slots != polled slots"
        assert got.min() >= 0 and got.max() + 8 <= 2 * lay.parity <= lay.region_bytes and not (got % 8).any()
        assert got.max() + 8 <= lay.counter


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("n16,two_shot", [(1, False), (513, False), (8 * 257, True), (8 * 257, False), (65536, True),
                                           (65536, False)])
def test_allreduce_pushes_meet_polls(world, n16, two_shot):
    if two_shot and n16 % world:
        pytest.skip("two-shot needs n16 % world == 0")
    lay = po.Layout(n16 * 16)                        # the largest message the region holds
    rng = np.random.default_rng(n16 + world)
    contrib = _rand_bits(rng, (world, n16 * 8), False)
    red = po.sum_in_rank_order(contrib, False)
    epoch = 7
    pushes = {s: po.allreduce_pushes(lay, s, world, epoch, po.words_of(contrib[s]), po.words_of(red), two_shot)
              for s in range(world)}
    polls = {r: po.allreduce_polls(lay, r, world, epoch, n16, two_shot) for r in range(world)}
    _check_meet(lay, world, pushes, polls)
    # the data a rank finds is its peers' contribution (one-shot) or slice / reduced slice (two-shot)
    off, data = po.polled_by(pushes, 0)
    assert len(off) == len(data)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("rows,hidden", [(1, 1024), (5, 8 * 8 * 97), (300, 8192)])
def test_norm_and_rs_gemm_pushes_meet_polls(world, rows, hidden):
    lay = po.Layout(rows * hidden * 2)
    rng = np.random.default_rng(rows * world)
    contrib = _rand_bits(rng, (world, rows, hidden), True)
    red = po.sum_in_rank_order(contrib, True)
    epoch = 0xFFFFFFFF
    pushes = {s: po.norm_pushes(lay, s, world, epoch, contrib[s], red) for s in range(world)}
    polls = {r: po.norm_polls(lay, r, world, epoch, rows, hidden) for r in range(world)}
    _check_meet(lay, world, pushes, polls)
    # the GEMM epilogue's push (rs_lane's address) is the norm kernel's scatter, word for word: the gather + norm kernel
    # finds what the unfused all-reduce + norm would have sent
    for s in range(world):
        rs = po.rs_gemm_pushes(lay, s, world, epoch, contrib[s])
        gather_only = po.norm_pushes(lay, s, world, epoch, contrib[s], red, pushed=True)
        for q in range(world):
            if q == s:
                continue
            full = dict(zip(*pushes[s][q]))
            rs_map = dict(zip(*rs[q]))
            area1 = set(gather_only[q][0])
            assert set(full) == set(rs_map) | area1 and not (set(rs_map) & area1)
            assert all(full[o] == d for o, d in rs_map.items())


@pytest.mark.parametrize("world", [2, 4, 8])
def test_argmax_pushes_meet_polls_and_combine(world):
    rows, vloc = 7, 101
    vtot = world * vloc - 5
    lay = po.Layout(rows * 16)
    rng = np.random.default_rng(world)
    full = orc.round_t(rng.standard_normal((rows, world * vloc)), False)
    full[1, :] = -np.inf
    full[2, 5] = np.nan
    full[3, :vtot] = np.nan
    full[4, vtot + 1] = 1e4                          # a padded column never counts
    full[5, vloc - 1] = full[5, vloc] = 9.0          # a tie across a rank boundary
    full[6, 3] = full[6, 7] = 9.0                    # a tie inside a rank
    pairs = [po.argmax_local(full[:, s * vloc:(s + 1) * vloc], s, vloc, vtot) for s in range(world)]
    pushes = {s: po.argmax_pushes(lay, s, world, 3, *pairs[s]) for s in range(world)}
    polls = {r: po.argmax_polls(lay, r, world, 3, rows) for r in range(world)}
    _check_meet(lay, world, pushes, polls)
    # the winner of the local winners (largest value, lowest index) is the argmax of the concatenated row
    vals = np.stack([p[0].view(np.float32) for p in pairs], 1).astype(np.float64)
    idx = np.stack([p[1] for p in pairs], 1).astype(np.int64)
    comb = []
    for v, i in zip(vals, idx):
        best = max(range(world), key=lambda s: (v[s], -i[s]))
        comb.append(i[best])
    exp = po.argmax_np(full[:, :vtot])
    assert np.array_equal(comb, exp)
    assert exp[1] == 0 and exp[3] == 0x7FFFFFFF and exp[5] == vloc - 1 and exp[6] == 3


@pytest.mark.parametrize("bf", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("world", [3, 4, 8])
def test_exact_sum_sees_own_contribution_first(world, bf):
    c = po.crafted_order_input(world, 64, bf)
    ref = po.sum_in_rank_order(c, bf)
    assert orc.from_bits(ref[:1], bf)[0] == (world - 2) * 2.0 ** -10
    for r in range(2, world):
        mut = po.sum_in_rank_order(c, bf, first=r)
        assert not np.array_equal(mut, ref), f"own-first at rank {r} gave the same bits"
    # ranks 0 and 1 add the same first two terms either way (fp32 addition commutes)
    for r in (0, 1):
        assert np.array_equal(po.sum_in_rank_order(c, bf, first=r), ref)


def test_norm_reference_sees_unrounded_sum():
    rng = np.random.default_rng(5)
    c = _rand_bits(rng, (4, 3, 256), False)
    res = _rand_bits(rng, (3, 256), False)
    g = orc.f64_to_bits(np.ones(256), False)
    _, stored, _, _ = po.allreduce_norm_ref(c, res, g, 1e-5, False)
    _, stored_mut, _, _ = po.allreduce_norm_ref(c, res, g, 1e-5, False, round_reduced=False)
    assert (stored != stored_mut).mean() > 0.05
