"""CPU tests of the shared-prefix attention's host side: ops.prefix_chunks on hand-built block tables, the argument checks of
b200_paged_decode_attn_prefix (reported, not crashed, before any CUDA call) and its export."""
import ctypes

import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200._lib import B200Error


def chunks(block_ids, lens, T, group):
    offs, rows, shared, mm = ops.prefix_chunks(torch.tensor(block_ids, dtype=torch.int32), torch.tensor(lens, dtype=torch.int32),
                                               T, group)
    o = offs.tolist()
    return [(rows.tolist()[a:b], s) for a, b, s in zip(o, o[1:], shared.tolist())], mm


def test_common_prefixes_of_different_lengths():
    T = 16
    tbl = [[1, 2, 3, 10, 0],      # group A: blocks 1 2 3 shared by rows 0, 2, 4
           [5, 6, 20, 0, 0],      # group B: blocks 5 6 shared by rows 1, 3
           [1, 2, 3, 11, 0],
           [5, 6, 21, 22, 0],
           [1, 2, 3, 12, 13]]
    lens = [60, 40, 50, 60, 70]
    got, mm = chunks(tbl, lens, T, 4)
    assert got == [([0, 2, 4], 48), ([1, 3], 32)] and mm == 3


def test_rows_need_not_be_adjacent_and_a_differing_block_ends_the_prefix():
    tbl = [[7, 8, 9, 1], [3, 4, 5, 6], [7, 8, 2, 0], [7, 8, 9, 4], [3, 4, 5, 6]]
    got, _ = chunks(tbl, [60, 63, 60, 60, 63], 16, 8)
    # group 7: rows 0, 2, 3 agree on blocks 7 8 only; group 3: rows 1, 4 on all four, capped at their lengths' whole blocks
    assert got == [([0, 2, 3], 32), ([1, 4], 48)]


def test_a_prefix_that_would_reach_a_members_last_token_is_capped():
    T = 16
    # identical tables: the block of each member's next token (position len) must never be shared
    got, _ = chunks([[1, 2, 3, 4]] * 3, [48, 47, 64], T, 4)
    assert got == [([0, 1, 2], 32)]      # row 1 holds 47 tokens: its third block is not whole, and takes the next token
    got, _ = chunks([[1, 2, 3, 4]] * 2, [32, 32], T, 4)
    assert got == [([0, 1], 32)]         # 32 cached: blocks 0-1 whole, the new token opens block 2
    got, _ = chunks([[1, 2]] * 2, [15, 40], T, 4)
    assert got == [([0], 0), ([1], 0)]   # a member with no whole block shares nothing: both rows run alone


def test_a_member_that_diverges_early_does_not_cut_the_others():
    T = 16
    tbl = [[1, 2, 3, 4, 5], [1, 2, 3, 4, 6], [1, 9, 9, 9, 9], [1, 2, 3, 4, 7], [1, 8, 8, 8, 8]]
    got, mm = chunks(tbl, [80] * 5, T, 4)
    # rows 0, 1, 3 share four blocks; rows 2 and 4 share only block 1 with them: fewer blocks saved as one group of five
    # (4 x 1) than as a group of three (2 x 4) and a group of two (1 x 1)
    assert got == [([0, 1, 3], 64), ([2, 4], 16)] and mm == 3
    got, _ = chunks([[1, 2, 3], [1, 2, 3], [1, 5, 6]], [40, 40, 10], T, 4)
    assert got == [([0, 1], 32), ([2], 0)]   # row 2 has no whole block cached: alone


def test_singletons_share_nothing():
    got, mm = chunks([[1, 2, 3], [4, 5, 6], [7, 8, 9]], [40, 40, 40], 16, 4)
    assert got == [([0], 0), ([1], 0), ([2], 0)] and mm == 1


@pytest.mark.parametrize("group", [1, 4, 8, 16])
def test_groups_larger_than_64_over_group_are_cut_into_chunks(group):
    cap = 64 // group
    n = 2 * cap + 3                        # two full chunks and a chunk of three
    tbl = [[9, 9, 100 + r] for r in range(n)] + [[5, 6, 7]]
    got, mm = chunks(tbl, [40] * n + [40], 16, group)
    want = [(list(range(c, min(c + cap, n))), 32) for c in range(0, n, cap)] + [([n], 0)]
    assert got == want and mm == cap
    for rows, _ in got:
        assert len(rows) * group <= 64


def test_a_chunk_of_one_left_after_the_cut_shares_nothing():
    n = 64 // 16 + 1                       # group 16: chunks of 4, and one row left
    got, _ = chunks([[3, 4, 100 + r] for r in range(n)], [40] * n, 16, 16)
    assert got == [([0, 1, 2, 3], 32), ([4], 0)]


def test_prefix_chunks_rejects_bad_inputs():
    good = torch.zeros(2, 3, dtype=torch.int32)
    lens = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(B200Error):
        ops.prefix_chunks(good.long(), lens, 16, 4)
    with pytest.raises(B200Error):
        ops.prefix_chunks(good, torch.zeros(3, dtype=torch.int32), 16, 4)
    with pytest.raises(B200Error):
        ops.prefix_chunks(good, lens, 16, 0)


def test_the_prefix_entry_is_exported_and_checks_its_arguments():
    lib = _lib.load()
    assert hasattr(lib, "b200_paged_decode_attn_prefix")
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def call(Hq=32, Hkv=8, D=128, B=8, chunks=2, members=4, offs=p, rows=p, shared=p, M=32, max_len=2048, T=64, q=p):
        return lib.b200_paged_decode_attn_prefix(q, 0, p, Hq, Hkv, D, B, chunks, members, offs, rows, shared, M, max_len, T, p, p,
                                                 p, 1.0, p, 4096, None)

    def err(**kw):
        assert call(**kw) == -1
        return lib.b200_last_error()
    assert b"null" in err(offs=None)
    assert b"null" in err(shared=None)
    assert b"chunks" in err(chunks=0)
    assert b"chunks" in err(chunks=9)
    assert b"max_members" in err(members=17)            # group 4 x 17 = 68 rows
    assert b"max_members" in err(members=0)
    assert b"grid" in err(Hkv=8, Hq=8, B=10000, chunks=9000, members=1)
    assert b"65535" in err(Hkv=1, Hq=1, B=70000, chunks=2, members=1)
    assert b"head_dim" in err(D=96)
    assert b"page_size" in err(T=48)
    assert b"multiple" in err(Hq=30)
    assert call(B=0) == 0                                # an empty batch launches nothing


def test_the_prefix_rule_follows_the_measured_boundary():
    from rtp_llm_b200.attention import prefix_rows_fit
    assert prefix_rows_fit(8, 32, 512, 4)         # 256 (chunk, kv head) pairs
    assert prefix_rows_fit(8, 16, 1024, 8)        # 128 pairs, half the context shared
    assert not prefix_rows_fit(8, 16, 512, 8)
    assert not prefix_rows_fit(8, 8, 1536, 8)     # 64 pairs: fewer, heavier CTAs lose
    assert not prefix_rows_fit(8, 64, 1536, 16)   # chunks of 16 rows


@pytest.mark.parametrize("kw", [dict(q_len=2), dict(beam_width=2), dict(tp_size=2, tp_rank=0), dict(q_len=2, tree=[-1, 0]),
                                dict(sampling="s")], ids=["q_len", "beam", "tp", "tree", "sampling"])
def test_the_shared_prefix_step_rejects_the_modes_it_does_not_cover(kw):
    import dataclasses

    from rtp_llm_b200.decode_step import TINY, SamplingParams, DecodeStep
    if kw.get("sampling") == "s":
        kw = dict(sampling=SamplingParams(temperature=0.8))
    with pytest.raises(ValueError, match="shared_prefix"):
        DecodeStep(dataclasses.replace(TINY, quant="int4"), 4, 100, torch.device("cpu"), shared_prefix=(2, 32), **kw)
