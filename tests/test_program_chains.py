"""CPU tests of tests/program_chains.py: the restated split-K plan on every branch, the restated ring depths, and what each chain
of tests/test_gpu_program_chains.py reaches in the persistent kernel (its name's claim, and the suite's coverage as a whole)."""
import pytest

from tests import program_chains as pc

GRID = 2 * pc.SMS     # 264 on an H100 SXM


@pytest.mark.parametrize("args,per", [
    ((1, 4, GRID, 16), 1),                          # want 1: every k-block its own CTA, S 4
    ((100, 8, GRID, 16), 4),                        # want 4 divides 8: S 2
    ((1, 12, GRID, 16), 3),                         # S 12 and 6 are not powers of two: d 3, S 4
    ((1, 32, GRID, 16), 2),                         # S 32 is above 16: d 2, S 16
    ((1, 600, GRID, 32), 75),                       # the first divisor from want up with S a power of two: S 8
    ((600, 2, GRID, 16), 6),                        # want 5 >= k_blocks: whole tiles, 3 per CTA
    ((1002, 32, GRID, 32), 128),                    # the lm_head: 4 whole tiles per CTA
    ((240, 7, GRID, 16), 7),                        # want 7 == k_blocks: one whole tile per CTA
    ((8, 16, GRID, 64, 8 * 16 * 64 * 128 * 4), 1),  # S 16 fits the workspace exactly
    ((8, 16, GRID, 64, 8 * 16 * 64 * 128 * 4 - 1), 2),   # one byte short: the next divisor, S 8
    ((8, 16, GRID, 64, 0), 16),                     # no room for any partial: whole tiles (the fallback)
    ((8, 16, 132, 64), 1),                          # half the grid: want 1 still
    ((100, 8, 132, 16), 8),                         # half the grid: want 7 -> d 8, whole tiles
])
def test_restated_sk_plan_takes_each_branch(args, per):
    assert pc.sk_plan(*args) == per


def test_restated_ring_depths_and_two_ctas_per_sm_everywhere():
    depths = {(f, b): (pc.seg_cfg(f, b)["WS"], pc.seg_cfg(f, b)["XS"]) for f in ("int4", "int8") for b in (16, 32, 64)}
    assert depths == {("int4", 16): (10, 4), ("int4", 32): (8, 4), ("int4", 64): (6, 3),
                      ("int8", 16): (5, 4), ("int8", 32): (4, 4), ("int8", 64): (3, 3)}
    # segment_inst.cuh static_asserts two CTAs per SM for every instance: no batch pad runs the kernel at 132 CTAs
    assert all(pc.seg_cfg(f, b)["per_sm"] == 2 for f in ("int4", "int8") for b in (16, 32, 64))
    assert {pc.segment_grid(f, b) for f in ("int4", "int8") for b in (16, 32, 64)} == {GRID}


def test_runs_tile_the_work_list_and_counters_advance_alike():
    """sk_range cuts the work list into consecutive runs; a CTA's counter after an op is its run length, for all three roles."""
    for nt, kb in ((1, 4), (600, 2), (8, 16), (240, 5)):
        per = pc.sk_plan(nt, kb, GRID, 16)
        runs = [pc.sk_run(nt, kb, per, c) for c in range(GRID)]
        covered = [k for g0, g1 in runs for k in range(g0, g1)]
        assert covered == list(range(nt * kb))
        # every CTA's run lies in one tile, or is a whole number of tiles
        for g0, g1 in runs:
            if g1 > g0:
                assert (g0 // kb == (g1 - 1) // kb) or (g0 % kb == 0 and g1 % kb == 0) or g1 == nt * kb


@pytest.mark.parametrize("chain", pc.CHAINS, ids=[c.name for c in pc.CHAINS])
def test_chain_reaches_what_its_name_claims(chain):
    cov = pc.coverage(chain, GRID)
    assert chain.claims, "a chain without a claim"
    for claim in chain.claims:
        assert pc.CLAIMS[claim](cov), f"{chain.name}: does not reach {claim!r}"
    assert cov == pc.coverage(chain), "the default grid is not 264"


def test_the_chains_cover_the_cross_op_machinery():
    covs = {c.name: pc.coverage(c, GRID) for c in pc.CHAINS}
    rings = [pc.mid_ring_phase1(c) for c in covs.values()]
    for ring in ("weight", "activation", "consumer"):
        assert any(r[ring] for r in rings), f"no op starts mid-{ring}-ring with phase 1"
    assert any(n > 250 for c in covs.values() for _, n in c["glue_after_idle"]), "no glue op after a GEMM leaving > 250 CTAs idle"
    assert any(all(pc.CLAIMS[k](c) for k in ("S16 then S2", "S2 then S4", "S4 then whole tiles")) for c in covs.values()), \
        "no chain runs S 16 -> S 2 -> S 4 -> whole tiles on one workspace"
    assert any(c["war"] for c in covs.values()), "no write-after-read chain"
    for k in ("several tiles per CTA", "segment break"):
        assert any(pc.CLAIMS[k](c) for c in covs.values()), k
    # batch pads 16 / 32 / 64, both dtypes, both persistent weight formats, and every glue op
    assert {pc.bpad_of(c.B) for c in pc.CHAINS} == {16, 32, 64}
    assert {c.B for c in pc.CHAINS} >= {1, 16, 17, 33, 64}
    assert {c.dtype for c in pc.CHAINS} == {"f16", "bf16"}
    assert {op.fmt for c in pc.CHAINS for op in c.ops if op.kind == "gemm"} == {"int4", "int8", "int8g"}
    assert {op.kind for c in pc.CHAINS for op in c.ops} == {"gemm", "norm", "rope", "embed", "table", "attn"}


def test_restated_recorder_breaks_segments_where_the_library_does():
    by_name = {c.name: c for c in pc.CHAINS}
    seg = lambda n: [len(s["ops"]) if "ops" in s else None for s in pc.segments(by_name[n])]
    assert seg("break int4 -> int8 gemm f16 b33") == [2, 1]                   # format change after the norm joined int4
    assert seg("break int8g gemm and hidden-9216 norm mid-chain f16 b16") == [1, None, None, 2]
    assert seg("break attention between rope and o gemm bf16 b17") == [2, None, 2]
    assert seg("glue-led table -> embedding -> norm -> gemm -> rope f16 b33") == [5]
    # a glue-only segment launches with the defaults of b200_program_launch
    s = pc.segments(by_name["glue-led table -> rope bf16 b17"])
    assert s == [{"ops": [0, 1], "key": (1, -1, -1), "bpad": 32, "fmt": "int4"}]


def test_buffer_roles():
    by_name = {c.name: c for c in pc.CHAINS}
    war = by_name["war gemm A->B, norm B->A, gemm A->B int4 bf16 b17"]
    assert pc.buffer_roles(war) == {"A": "in", "B": "out", "res": "in"}
    assert pc.written(war) == ["B", "A", "res"]
    glue = by_name["glue-led table -> embedding -> norm -> gemm -> rope f16 b33"]
    assert pc.buffer_roles(glue)["pl"] == "out"          # written by the block-table op before the rope reads it
    assert pc.buffer_roles(by_name["glue-led table -> rope bf16 b17"])["qkv"] == "in"
