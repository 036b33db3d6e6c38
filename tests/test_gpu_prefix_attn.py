"""GPU tests of b200_paged_decode_attn_prefix: rows of different requests that share leading pages grouped into chunks, each
chunk's shared pages read once.

The op is b200_paged_decode_attn on the batch's rows, so the float64 reference and its error budget are those of the plain
kernel. The exact properties pin the row indirection: sharing never changes a bit within a chunking; contiguous uniform chunks
are the beam kernel and one row per chunk is the plain kernel, bit for bit; nothing of another member, and no value of the
chunk arrays, reaches a row's output or anything outside `out`."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests import pdl_cases as pc  # noqa: E402
from tests.test_gpu_pdl_hazards import _run_case  # noqa: E402

DEV = torch.device("cuda:0")
SPLITS = "B200_ATTN_TILES_PER_SPLIT"


class Case:
    """groups: one (shared tokens, [each member's length with its new token]) per group of requests. shared is a multiple of
    the page size T; the members point at the same pages over it and at pages of their own after it. The members of all groups
    are scattered over the batch by a seeded permutation, so a group's rows are not adjacent."""

    def __init__(self, Hq, Hkv, T, D, groups, dtype, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.T, self.dtype = T, dtype
        lens = [L for _, ls in groups for L in ls]
        B = len(lens)
        M = max(math.ceil(L / T) for L in lens)
        npages = 1 + sum(s // T + sum(math.ceil(L / T) - s // T for L in ls) for s, ls in groups)
        self.pool = torch.randn(npages, 2, Hkv, T, D, generator=g).to(dtype)
        self.q = torch.randn(B, Hq, D, generator=g).to(dtype)
        it = iter((torch.randperm(npages - 1, generator=g) + 1).tolist())
        perm = torch.randperm(B, generator=g).tolist()        # member k of the listing sits at row perm[k]
        self.block_ids = torch.zeros(B, M, dtype=torch.int32)
        self.seq = torch.zeros(B, dtype=torch.int32)
        self.own = {}                                         # row -> its private page ids
        self.members, k = [], 0
        for s, ls in groups:
            common = [next(it) for _ in range(s // T)]
            rows = []
            for L in ls:
                r = perm[k]
                k += 1
                mine = [next(it) for _ in range(math.ceil(L / T) - s // T)]
                self.block_ids[r, :len(common) + len(mine)] = torch.tensor(common + mine, dtype=torch.int32)
                self.seq[r] = L - 1
                self.own[r] = mine
                rows.append(r)
            self.members.append((s, rows))
        self.max_len = int(self.seq.max()) + 1

    def chunks(self, cap, shared=None):
        """The groups cut into chunks of at most cap rows, each with its group's shared length (or `shared`, one per chunk),
        and the largest chunk's row count as max_members."""
        offs, rows, sh = [0], [], []
        for s, rs in self.members:
            for c in range(0, len(rs), cap):
                rows += rs[c:c + cap]
                offs.append(len(rows))
                sh.append(s)
        if shared is not None:
            sh = shared
        i32 = dict(dtype=torch.int32)
        return torch.tensor(offs, **i32), torch.tensor(rows, **i32), torch.tensor(sh, **i32), max(np.diff(offs))


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def run_prefix(c: Case, chunking, pool=None, guarded=False, out_init=None):
    offs, rows, sh, max_members = chunking
    B, Hq, D = c.q.shape
    pool = c.pool if pool is None else pool
    ws = ops.attn_workspace(B, Hq, pool.shape[2], c.max_len, DEV)
    buf, out = probe.guarded_empty((B, Hq * D), c.q.dtype)
    if out_init is not None:
        out.copy_(out_init)
    ops.paged_decode_attn_prefix(c.q.to(DEV), pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV)), c.seq.to(DEV),
                                 offs.to(DEV), rows.to(DEV), sh.to(DEV), int(max_members), c.max_len, ws, out=out)
    torch.cuda.synchronize()
    return (out, buf) if guarded else out.clone()


def run_rows(c: Case, pool=None):
    B, Hq, D = c.q.shape
    pool = c.pool if pool is None else pool
    ws = ops.attn_workspace(B, Hq, pool.shape[2], c.max_len, DEV)
    out = ops.paged_decode_attn(c.q.to(DEV), pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV)), c.seq.to(DEV),
                                c.max_len, ws)
    torch.cuda.synchronize()
    return out


def _tail(P, n, step, first=1):
    return [P + first + step * i for i in range(n)]


# name, D, Hq, Hkv, T, groups (shared tokens, member lengths), dtype, env. The shared lengths are whole pages but (mostly) not
# whole 64-token tiles, the member lengths ragged.
CASES = [
    ("g4 p16 d128", 128, 8, 2, 16, [(272, _tail(272, 5, 13)), (48, [49, 200, 60]), (0, [90])], torch.float16, None),
    ("g8 p64 bf16 cluster merge", 128, 16, 2, 64, [(320, _tail(320, 8, 9)), (128, [129, 300])], torch.bfloat16, {SPLITS: 2}),
    ("g2 p128 d64 workspace merge", 64, 4, 2, 128, [(640, [700, 641, 650, 900, 660, 777]), (0, [20, 300])], torch.float16,
     {SPLITS: 1}),
    ("g1 p32 d256", 256, 4, 4, 32, [(160, _tail(160, 12, 7)), (96, [97, 130])], torch.float16, None),
    ("g6 p32 bf16 d128", 128, 12, 2, 32, [(224, _tail(224, 10, 11, 3)), (32, [33, 64, 65])], torch.bfloat16, None),
    ("g3 p16 d256 workspace merge", 256, 6, 2, 16, [(400, _tail(400, 7, 31)), (16, [17, 18])], torch.bfloat16, {SPLITS: 1}),
    ("g5 p64 d64 cluster merge", 64, 10, 2, 64, [(576, _tail(576, 4, 50)), (192, _tail(192, 9, 3))], torch.float16, {SPLITS: 1}),
    ("g7 p128 d128", 128, 7, 1, 128, [(256, _tail(256, 9, 40)), (0, [5, 6])], torch.float16, None),
]
IDS = [c[0] for c in CASES]


def _case(case, seed):
    _, D, Hq, Hkv, T, groups, dtype, env = case
    return Case(Hq, Hkv, T, D, groups, dtype, seed=seed), env, 64 // (Hq // Hkv)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_sharing_never_changes_a_bit(case):
    """Every row has the bits of the same launch with shared_lengths all 0, whatever is declared within the caller's contract
    (any value up to the pages the members share; the kernel rounds it down to whole 64-token tiles) and for negative values."""
    c, env, cap = _case(case, 1)
    P = c.chunks(cap)[2].tolist()
    with probe.env_set(env):
        base = run_prefix(c, c.chunks(cap, [0] * len(P)))
        for sh in (P, [min(64, p) for p in P], [min(100, p) for p in P], [max(p - 1, 0) for p in P], [-3] * len(P)):
            assert same_bits(run_prefix(c, c.chunks(cap, sh)), base), f"shared_lengths {sh} changed the output"


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_one_row_per_chunk_is_the_plain_kernel(case):
    c, env, _ = _case(case, 2)
    B = c.q.shape[0]
    order = torch.randperm(B, generator=torch.Generator().manual_seed(5)).to(torch.int32)
    one = (torch.arange(B + 1, dtype=torch.int32), order, torch.zeros(B, dtype=torch.int32), 1)
    with probe.env_set(env):
        assert same_bits(run_prefix(c, one), run_rows(c))


BEAM_LIKE = [("g4 W4 p16", 128, 8, 2, 16, 4, torch.float16, None), ("g8 W8 p64 bf16", 128, 16, 2, 64, 8, torch.bfloat16, {SPLITS: 2}),
             ("g2 W6 d64 p128 workspace merge", 64, 4, 2, 128, 6, torch.float16, {SPLITS: 1}),
             ("g1 W16 d256 p32", 256, 4, 4, 32, 16, torch.float16, None)]


@pytest.mark.parametrize("case", BEAM_LIKE, ids=[c[0] for c in BEAM_LIKE])
def test_contiguous_uniform_chunks_are_the_beam_kernel(case):
    _, D, Hq, Hkv, T, W, dtype, env = case
    g = torch.Generator().manual_seed(3)
    R = 3
    shared = [T * 5, T * 2, 0]
    groups = [(s, [s + 1 + int(x) for x in torch.randint(0, 150, (W,), generator=g)]) for s in shared]
    c = Case(Hq, Hkv, T, D, groups, dtype, seed=4)
    # renumber rows so that request b's members are rows b * W + i, as the beam kernel takes them
    order = [r for _, rs in c.members for r in rs]
    inv = torch.tensor(order)
    c.q, c.block_ids, c.seq = c.q[inv], c.block_ids[inv], c.seq[inv]
    i32 = dict(dtype=torch.int32)
    chunking = (torch.arange(0, R * W + 1, W, **i32), torch.arange(R * W, **i32), torch.tensor(shared, **i32), W)
    ws = ops.attn_workspace(R * W, Hq, Hkv, c.max_len, DEV)
    with probe.env_set(env):
        got = run_prefix(c, chunking)
        beam = ops.paged_decode_attn_beam(c.q.view(R, W, Hq, D).to(DEV), c.pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV)),
                                          c.seq.to(DEV), chunking[2].to(DEV), c.max_len, ws)
        torch.cuda.synchronize()
    assert same_bits(got, beam.view(R * W, -1))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_prefix_attention_within_the_error_budget(case):
    """Against the float64 reference of the rows within the attention error budget, nothing written outside the output. The
    cases with SPLITS set force the cluster merge (2..8 splits) or the workspace merge (more)."""
    name = case[0]
    c, env, cap = _case(case, 5)
    with probe.env_set(env):
        out, buf = run_prefix(c, c.chunks(cap), guarded=True)
    probe.RESULTS.clear()
    B, Hq, D = c.q.shape
    f64, E = orc.paged_decode_attn_np(c.q.float().numpy(), c.pool.float().numpy(), c.block_ids.numpy(), c.seq.numpy(), c.T,
                                      with_abs=True)
    ok, info = probe.budget_info(out, f64, E, c.dtype == torch.bfloat16)
    probe.report(name + " [prefix kernel vs float64, error budget]", ok, info)
    probe.report_bands(name, buf)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad


@pytest.mark.parametrize("fill", [3.0e4, float("nan")], ids=["large", "nan"])
@pytest.mark.parametrize("case", CASES[:3], ids=IDS[:3])
def test_a_members_own_pages_reach_no_other_row(case, fill):
    c, env, cap = _case(case, 6)
    ch = c.chunks(cap)
    T = c.T
    with probe.env_set(env):
        clean = run_prefix(c, ch)
        pool = c.pool.clone()
        for r, L in enumerate((c.seq + 1).tolist()):          # the slots past every row's length, inside its last page
            if L % T:
                pool[c.block_ids[r, (L - 1) // T].item(), :, :, L % T:, :] = fill
        assert same_bits(run_prefix(c, ch, pool=pool), clean), "slots past a row's length reached an output"
        B = c.q.shape[0]
        for r in list(c.own)[::3]:
            if not c.own[r]:
                continue
            dirty = pool.clone()
            dirty[torch.tensor(c.own[r])] = fill
            out = run_prefix(c, ch, pool=dirty)
            keep = [k for k in range(B) if k != r]
            assert same_bits(out[keep], clean[keep]), f"row {r}'s pages reached another row"


def test_bad_chunk_data_stays_inside_out():
    """Rows in no chunk keep their bytes; an out-of-range row index is skipped; a chunk longer than max_members is cut off;
    offsets out of order or out of range are clamped. Every value passed is a valid int32 the kernel must clamp: nothing is
    read or written outside q, out and the page list, and the rows it does write have their bits from a clean chunking."""
    c, env, cap = _case(CASES[0], 7)
    B, Hq, D = c.q.shape
    s, rows0 = c.members[0]                                  # 5 rows of the 9
    assert len(rows0) == 5 and B == 9
    i32 = dict(dtype=torch.int32)
    marker = torch.full((B, Hq * D), 7.0, dtype=c.dtype, device=DEV)
    # clean reference: the group's first 3 rows as one chunk, max_members 3, and three empty chunks (the same split plan)
    ref = run_prefix(c, (torch.tensor([0, 3, 3, 3, 3], **i32), torch.tensor(rows0[:3] + [0] * (B - 3), **i32),
                         torch.tensor([s, 0, 0, 0], **i32), 3))
    listed = set(rows0[:3])
    # the group's 5 rows in one chunk (two past max_members 3); a chunk of rows outside [0, B) up to an offset past the
    # batch; offsets that run backwards and below 0
    rows = rows0 + [-1, B, 1 << 30, rows0[4]]
    offs = torch.tensor([0, 5, 1 << 30, -5, -7], **i32)
    out, buf = run_prefix(c, (offs, torch.tensor(rows, **i32), torch.tensor([s, 1 << 20, 64, -1], **i32), 3), guarded=True,
                          out_init=marker)
    probe.RESULTS.clear()
    probe.report_bands("bad chunk data", buf)
    assert all(ok for _, ok in probe.RESULTS), probe.RESULTS
    for r in range(B):
        if r in listed:
            assert same_bits(out[r], ref[r]), f"row {r}"
        else:
            assert same_bits(out[r], marker[r]), f"row {r} is in no chunk (or past max_members) but was written"


def test_graph_replay_with_updated_lengths():
    """Captured once, replayed as the lengths advance in place: every replay gives the bits of an eager call on the same state."""
    c, _, cap = _case(CASES[0], 8)
    B, Hq, D = c.q.shape
    c.block_ids = torch.cat([c.block_ids, torch.zeros(B, 1, dtype=torch.int32)], 1)   # room for the lengths to grow (page 0)
    offs, rows, sh, _ = [t.to(DEV) if torch.is_tensor(t) else t for t in c.chunks(cap)]
    q, pool, pl = c.q.to(DEV), c.pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV))
    max_len = c.max_len + 4          # (four more tokens stay within every row's last page or the table's zero-padded column)
    ws = ops.attn_workspace(B, Hq, c.pool.shape[2], max_len, DEV)
    seq_g, seq_e = c.seq.to(DEV), c.seq.to(DEV)
    out_g, out_e = (torch.empty(B, Hq * D, dtype=c.dtype, device=DEV) for _ in range(2))
    call = lambda seq, out: ops.paged_decode_attn_prefix(q, pool, pl, seq, offs, rows, sh, cap, max_len, ws, out=out)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(seq_g, out_g)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(seq_g, out_g)
    for step in range(3):
        out_g.zero_()
        graph.replay()
        call(seq_e, out_e)
        torch.cuda.synchronize()
        assert same_bits(out_g, out_e), f"replay {step}"
        seq_g.add_(1)
        seq_e.add_(1)


def _pdl_prefix(dtype, B=7, Hq=8, Hkv=2, T=16, D=128, max_len=200, members=3):
    """A pdl_cases-style case of the prefix entry point: rows in chunks of up to `members`, scattered over the batch, whose
    page-list rows share their first pages; every dynamic input (pages, lengths, chunking) changes between versions."""
    M = -(-max_len // T)
    P = B * 2 * M + 1

    def dyn(seed):
        g = pc._gen(seed)
        pl = pc._page_list(g, B, M, P)
        seq = torch.randint(max_len - 64, max_len, (B,), generator=g, dtype=pc.I32)
        rows = torch.randperm(B, generator=g).to(pc.I32)
        offs = list(range(0, B, members)) + [B]
        shared = []
        for a, b in zip(offs, offs[1:]):
            rs = rows[a:b].tolist()
            s = T * (int(seq[rs].min()) // T) - T * int(torch.randint(0, 3, (1,), generator=g))
            shared.append(max(s, 0))
            for r in rs[1:]:
                pl[r, :, :, :s // T] = pl[rs[0], :, :, :s // T]
        return dict(q=pc._randn(g, B, Hq, D, dtype=dtype), pool=pc._randn(g, P, 2, Hkv, T, D, dtype=dtype), pl=pl,
                    seq=seq.to(pc.DEV), offs=torch.tensor(offs, dtype=pc.I32, device=pc.DEV), rows=rows.to(pc.DEV),
                    shared=torch.tensor(shared, dtype=pc.I32, device=pc.DEV))

    def call(b):
        ops.paged_decode_attn_prefix(b["q"], b["pool"], b["pl"], b["seq"], b["offs"], b["rows"], b["shared"], members, max_len,
                                     b["ws"], out=b["out"])

    def setup():
        ws = ops.attn_workspace(B, Hq, Hkv, max_len, pc.DEV).numel()
        return pc.Spec(dyn, call, outs={"out": ((B, Hq * D), dtype)}, ws={"ws": (ws, -(-B * Hkv * 4 // 256) * 256)})
    return setup


PDL = [pc.Case("attn prefix cluster merge bf16", ("paged_decode_attn_kernel",), _pdl_prefix(pc.BF16), pc.CLUSTER),
       pc.Case("attn prefix workspace merge f16", ("paged_decode_attn_kernel",), _pdl_prefix(pc.F16, max_len=900), pc.WORKSPACE)]


@pytest.mark.parametrize("case", PDL, ids=[c.name for c in PDL])
def test_prefix_entry_waits_for_its_grid_dependency(case):
    _run_case(case)


# ------------------------------------------------------------------------------------------------ the decode step
def _forced_step(prefix: bool):
    from rtp_llm_b200.decode_step import DecodeStep

    class Forced(DecodeStep):
        """The shared-prefix step with its attention forced (the tiny batches here are below attention.prefix_rows_fit)."""

        def upload_inputs(self):
            super().upload_inputs()
            self.use_prefix = prefix
    return Forced


@pytest.mark.parametrize("mode", ["eager", "graph", "graph+pdl"])
@pytest.mark.parametrize("quant,n,prefix", [("int4", 4, 96), ("f16", 3, 40)], ids=["int4 groups of 4", "f16 groups of 3"])
def test_shared_prefix_step_against_the_step_oracle(quant, n, prefix, mode):
    """DecodeStep(shared_prefix=(n, prefix)) on the prefix kernel: the groups' rows are scattered over the batch, share the
    whole pages of the prefix every member has cached, and prefix_chunks finds them. Logits against the step oracle, and
    within its tolerance of the same step on the per-row kernel."""
    import dataclasses

    from rtp_llm_b200.decode_step import TINY
    from tests.step_oracle import check_logits, device_state, oracle_step
    from tests.step_oracle import bits as step_bits
    cfg = dataclasses.replace(TINY, quant=quant)
    T, B = cfg.tokens_per_block, 12
    kw = dict(keep_reference=True, ragged=True, seed=5, pdl="pdl" in mode, shared_prefix=(n, prefix))
    new, old = _forced_step(True)(cfg, B, 160, DEV, **kw), _forced_step(False)(cfg, B, 160, DEV, **kw)
    calls = []
    orig = ops.paged_decode_attn_prefix
    offs, rows, shared, mm = (t.cpu() if torch.is_tensor(t) else t for t in new.chunks)
    groups = [rows[a:b].tolist() for a, b in zip(offs.tolist(), offs.tolist()[1:])]
    assert mm == n and any(len(g) > 1 and g != list(range(g[0], g[0] + len(g))) for g in groups), groups
    tbl = new.block_ids_h
    for g, s in zip(groups, shared.tolist()):
        assert s == (0 if len(g) == 1 else min([prefix // T] + [int(new.seq_lens_h[r]) // T for r in g]) * T)
        assert all(torch.equal(tbl[r, :s // T], tbl[g[0], :s // T]) for r in g)
    assert shared.max() > 0
    try:
        if "graph" in mode:
            new.capture()
            old.capture()
        state, kv_before = device_state(new), [step_bits(L["kv"]) for L in new.layers]
        n0 = ops.launch_count()
        ops.paged_decode_attn_prefix = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
        for m in (new, old):
            m.replay() if "graph" in mode else m.run()
        torch.cuda.synchronize()
        if mode == "eager":                  # (a graph replay launches outside the library's count)
            assert ops.launch_count() > n0
            assert len(calls) == cfg.layers      # the prefix kernel in every layer of the new step, never in the old
        check_logits(new.logits.float().cpu().numpy(), oracle_step(state, kv_before))
        check_logits(new.logits.float().cpu().numpy(), old.logits.float().cpu().numpy())
    finally:
        ops.paged_decode_attn_prefix = orig
        ops.set_pdl(False)


def test_shared_prefix_step_is_no_decode_program():
    import dataclasses

    from rtp_llm_b200.decode_step import TINY, DecodeStep
    model = DecodeStep(dataclasses.replace(TINY, quant="int4"), 4, 100, DEV, shared_prefix=(2, 32))
    with pytest.raises(ValueError, match="shared-prefix"):
        model.build_program()
