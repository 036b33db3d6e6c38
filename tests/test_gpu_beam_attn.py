"""GPU tests of b200_paged_decode_attn_beam: the attention of a request's beams in one CTA, reading the K/V they share once.

Semantically the op is b200_paged_decode_attn on the requests * beam_width rows, so the float64 reference and its error budget
are those of the plain kernel. What pins the new code are exact properties: beam_width 1 is the plain kernel bit for bit; the
shared length a caller declares never changes a bit; nothing a beam owns reaches another beam's output."""
import dataclasses
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops, rope  # noqa: E402
from rtp_llm_b200.attention import beam_rows_fit  # noqa: E402
from rtp_llm_b200.decode_step import TINY, TINY_QWEN3, DecodeStep  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests.step_oracle import check_logits, device_state, oracle_step  # noqa: E402
from tests.step_oracle import bits as step_bits  # noqa: E402

DEV = torch.device("cuda:0")
SPLITS = "B200_ATTN_TILES_PER_SPLIT"


class PerRowBeamStep(DecodeStep):
    """The beam step with the attention it had before the beam kernel: b200_paged_decode_attn on every beam's row."""

    def _attention(self, L):
        ops.paged_decode_attn(self.q, L["kv"], self.page_list, self.seq_lens, self.ctx, self.attn_ws, out=self.attn)


@dataclasses.dataclass
class Case:
    q: torch.Tensor           # [B, W, Hq, D]
    pool: torch.Tensor        # [P, 2, Hkv, T, D]
    block_ids: torch.Tensor   # [B*W, M]
    seq: torch.Tensor         # [B*W] tokens cached before the new one
    shared: torch.Tensor      # [B] tokens every beam of the request shares (whole pages)
    own: list                 # per row: the page ids no other row points at


def make_case(Hq, Hkv, T, D, W, requests, dtype, seed=0, extra_pages=0):
    """requests: one (shared tokens, [each beam's length with its new token]) per request. shared is a multiple of the page
    size T: the request's beams point at the same pages over it and at pages of their own after it. extra_pages: page-table
    columns beyond the longest sequence (room to grow, or a max_seq_len looser than the lengths); they point at page 0."""
    g = torch.Generator().manual_seed(seed)
    B = len(requests)
    assert all(s % T == 0 and len(lens) == W and min(lens) > s for s, lens in requests)
    M = max(math.ceil(max(lens) / T) for _, lens in requests) + extra_pages
    npages = 1 + sum(s // T + sum(math.ceil(L / T) - s // T for L in lens) for s, lens in requests)
    pool = torch.randn(npages, 2, Hkv, T, D, generator=g).to(dtype)
    q = torch.randn(B, W, Hq, D, generator=g).to(dtype)
    it = iter((torch.randperm(npages - 1, generator=g) + 1).tolist())
    block_ids = torch.zeros(B * W, M, dtype=torch.int32)
    own = []
    for b, (s, lens) in enumerate(requests):
        common = [next(it) for _ in range(s // T)]
        for i, L in enumerate(lens):
            mine = [next(it) for _ in range(math.ceil(L / T) - s // T)]
            block_ids[b * W + i, :len(common) + len(mine)] = torch.tensor(common + mine, dtype=torch.int32)
            own.append(mine)
    seq = torch.tensor([L - 1 for _, lens in requests for L in lens], dtype=torch.int32)
    return Case(q, pool, block_ids, seq, torch.tensor([s for s, _ in requests], dtype=torch.int32), own)


def run_beam(c: Case, shared=None, pool=None, max_len=None, guarded=False):
    B, W, Hq, D = c.q.shape
    pool = c.pool if pool is None else pool
    max_len = max_len or int(c.seq.max()) + 1
    ws = ops.attn_workspace(B * W, Hq, pool.shape[2], max_len, DEV)
    buf, out = probe.guarded_empty((B, W, Hq * D), c.q.dtype)
    sh = (c.shared if shared is None else torch.tensor(shared, dtype=torch.int32)).to(DEV)
    ops.paged_decode_attn_beam(c.q.to(DEV), pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV)), c.seq.to(DEV), sh, max_len, ws,
                               out=out)
    torch.cuda.synchronize()
    return (out, buf) if guarded else out.clone()


def run_rows(c: Case, pool=None, max_len=None):
    """b200_paged_decode_attn on the B * W rows of the same tables."""
    B, W, Hq, D = c.q.shape
    pool = c.pool if pool is None else pool
    max_len = max_len or int(c.seq.max()) + 1
    ws = ops.attn_workspace(B * W, Hq, pool.shape[2], max_len, DEV)
    out = ops.paged_decode_attn(c.q.view(B * W, Hq, D).to(DEV), pool.to(DEV), ops.convert_block_table(c.block_ids.to(DEV)),
                                c.seq.to(DEV), max_len, ws)
    torch.cuda.synchronize()
    return out.view(B, W, Hq * D)


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


# ------------------------------------------------------------------------------------------------ 1. beam_width 1
WIDTH_ONE = [
    ("g4 p64", 128, 8, 2, 64, [300, 64, 65, 1], torch.float16, None),
    ("g8 p16 bf16 cluster merge", 128, 16, 2, 16, [130, 700, 17], torch.bfloat16, {SPLITS: 2}),
    ("g16 workspace merge", 128, 16, 1, 32, [900, 70], torch.float16, {SPLITS: 1}),
    ("d64 mha p32", 64, 4, 4, 32, [64, 65, 190], torch.float16, None),
    ("d256 g32 p128", 256, 32, 1, 128, [127, 300], torch.float16, None),
    ("g64 bf16", 128, 64, 1, 64, [200, 3], torch.bfloat16, None),
]


@pytest.mark.parametrize("case", WIDTH_ONE, ids=[c[0] for c in WIDTH_ONE])
def test_width_one_is_the_plain_kernel_bit_for_bit(case):
    """One beam per request and nothing shared: the same plan, row tiles and operation order as b200_paged_decode_attn."""
    _, D, Hq, Hkv, T, lens, dtype, env = case
    c = make_case(Hq, Hkv, T, D, 1, [(0, [L]) for L in lens], dtype, seed=2)
    with probe.env_set(env):
        assert same_bits(run_beam(c), run_rows(c))


# ------------------------------------------------------------------------------------------------ 2. sharing keeps the bits
SHARING = [
    # name, D, Hq, Hkv, T, W, requests (shared tokens, lengths), dtype, env
    ("g4 W4 p16", 128, 8, 2, 16, 4, [(256, [300, 257, 290, 330]), (128, [129, 200, 140, 150])], torch.float16, None),
    ("g8 W8 p64 bf16 cluster merge", 128, 16, 2, 64, 8, [(320, [321 + 9 * i for i in range(8)])], torch.bfloat16, {SPLITS: 2}),
    ("g2 W6 p128 d64 workspace merge", 64, 4, 2, 128, 6, [(640, [700, 641, 650, 900, 660, 777])], torch.float16, {SPLITS: 1}),
    ("g4 W16 p32 d256", 256, 4, 1, 32, 16, [(192, [200 + 7 * i for i in range(16)])], torch.float16, None),
]


@pytest.mark.parametrize("case", SHARING, ids=[c[0] for c in SHARING])
def test_the_declared_shared_length_never_changes_a_bit(case):
    """On tables whose beams share P tokens, every shared_lengths from 0 to P gives the same bits: a row meets the tiles of
    its sequence in the same order either way, and the other beams' stages leave it untouched. Values that are no multiple
    of 64 or of the page size, negative, or beyond the shortest beam are rounded down and clamped, not trusted (in these
    cases the shortest beam ends less than a tile past P, so every value is within the caller's contract)."""
    _, D, Hq, Hkv, T, W, requests, dtype, env = case
    c = make_case(Hq, Hkv, T, D, W, requests, dtype, seed=3)
    with probe.env_set(env):
        base = run_beam(c, shared=[0] * len(requests))
        P = [s for s, _ in requests]
        tries = [[min(k, p) for p in P] for k in range(64, max(P) + 1, 64)]
        assert all((min(lens) - 1) // 64 * 64 <= p for p, lens in requests)
        tries += [P, [p - 1 for p in P], [17] * len(P), [100] * len(P), [-5] * len(P), [p + 30 for p in P], [1 << 20] * len(P)]
        for sh in tries:
            assert same_bits(run_beam(c, shared=sh), base), f"shared_lengths {sh} changed the output"
        # and what they are the bits of: the plain kernel's answer on the same rows, within its documented tolerance
        tol = 2e-2 if dtype == torch.bfloat16 else 1e-2
        np.testing.assert_allclose(base.float().cpu().numpy(), run_rows(c).float().cpu().numpy(), rtol=tol, atol=tol)


# ------------------------------------------------------------------------------------------------ 3. isolation
@pytest.mark.parametrize("fill", [3.0e4, float("nan")], ids=["large", "nan"])
@pytest.mark.parametrize("case", SHARING[:3], ids=[c[0] for c in SHARING[:3]])
def test_a_beams_own_pages_reach_no_other_beam(case, fill):
    _, D, Hq, Hkv, T, W, requests, dtype, env = case
    c = make_case(Hq, Hkv, T, D, W, requests, dtype, seed=4)
    with probe.env_set(env):
        clean = run_beam(c)
        # the slots past every beam's length, inside its last page, are nobody's
        pool = c.pool.clone()
        for r, L in enumerate((c.seq + 1).tolist()):
            if L % T:
                pool[c.block_ids[r, (L - 1) // T].item(), :, :, L % T:, :] = fill
        assert same_bits(run_beam(c, pool=pool), clean), "slots past a beam's length reached an output"
        for k in range(0, len(c.own), max(W - 1, 1)):       # a beam of every request, at varying beam indices
            dirty = pool.clone()
            dirty[torch.tensor(c.own[k])] = fill
            out = run_beam(c, pool=dirty).view(len(c.own), -1)
            keep = [r for r in range(len(c.own)) if r != k]
            assert same_bits(out[keep], clean.view(len(c.own), -1)[keep]), f"beam row {k}'s pages reached another beam"


# ------------------------------------------------------------------------------------------------ 4. budget across shapes
def _tail(P, W, step, first=1):
    return [P + first + step * i for i in range(W)]


BUDGET = [
    # name, D, Hq, Hkv, T, W, requests, dtype, env, max_len
    ("rows 16 g4 W4 p64", 128, 8, 2, 64, 4, [(1984, _tail(1984, 4, 9, 29)), (64, _tail(64, 4, 1))], torch.float16, None, None),
    ("rows 32 g4 W8 p16 bf16", 128, 8, 2, 16, 8, [(256, _tail(256, 8, 31)), (0, _tail(0, 8, 40, 5))], torch.bfloat16, None, None),
    ("rows 64 g4 W16 p32", 128, 4, 1, 32, 16, [(128, _tail(128, 16, 23))], torch.float16, None, None),
    ("rows 64 g8 W8 p128", 128, 16, 2, 128, 8, [(512, _tail(512, 8, 57, 3)), (128, _tail(128, 8, 64, 64))], torch.float16, None, None),
    ("rows 12 g4 W3 d64 p16", 64, 8, 2, 16, 3, [(192, [193, 400, 258]), (64, [70, 65, 66])], torch.float16, None, None),
    ("rows 24 g8 W3 d256 p64 bf16", 256, 16, 2, 64, 3, [(128, [129, 300, 200])], torch.bfloat16, None, None),
    ("rows 2 mha W2 p32", 128, 4, 4, 32, 2, [(64, [65, 250]), (0, [1, 2])], torch.float16, None, None),
    ("rows 16 g1 W16 d64 bf16", 64, 2, 2, 64, 16, [(64, _tail(64, 16, 13))], torch.bfloat16, None, None),
    ("all but the new token shared", 128, 8, 2, 64, 4, [(256, [257] * 4), (128, [129] * 4)], torch.float16, None, None),
    ("nothing shared, ring wraps", 128, 8, 2, 16, 4, [(0, [300, 17, 129, 260])], torch.float16, None, None),
    ("cluster merge 2 splits", 128, 8, 2, 64, 4, [(64, _tail(64, 4, 5)), (0, _tail(0, 4, 30))], torch.float16, {SPLITS: 1}, None),
    ("cluster merge 8 splits d64 bf16", 64, 8, 2, 32, 4, [(448, _tail(448, 4, 20)), (64, [65, 70, 200, 66])], torch.bfloat16,
     {SPLITS: 1}, None),
    ("cluster merge 5 splits rows 64", 128, 16, 2, 64, 8, [(512, _tail(512, 8, 11))], torch.float16, {SPLITS: 2}, None),
    ("workspace merge 15 splits", 128, 8, 2, 16, 4, [(768, _tail(768, 4, 60)), (128, [129, 900, 130, 500])], torch.float16,
     {SPLITS: 1}, None),
    ("workspace merge rows 64 d256", 256, 8, 1, 64, 8, [(576, _tail(576, 8, 17))], torch.float16, {SPLITS: 1}, None),
    ("max_seq_len 4096", 128, 8, 2, 64, 4, [(256, _tail(256, 4, 100))], torch.float16, None, 4096),
    ("longer than max_seq_len", 128, 8, 2, 64, 4, [(256, [300, 500, 257, 420]), (384, [400, 390, 385, 500])], torch.float16, None,
     320),
]


@pytest.mark.parametrize("case", BUDGET, ids=[c[0] for c in BUDGET])
def test_beam_attention_within_the_error_budget(case):
    """Against the float64 reference of the B * W rows within the attention error budget, against the plain kernel on those
    rows within its documented tolerance, and nothing written outside the output. A sequence longer than max_seq_len is cut
    at the split plan's bound, as the plain kernel cuts it: there the plain kernel alone is the reference."""
    name, D, Hq, Hkv, T, W, requests, dtype, env, max_len = case
    extra = 0 if max_len is None else max(0, math.ceil(max_len / T) - math.ceil(max(max(l) for _, l in requests) / T))
    c = make_case(Hq, Hkv, T, D, W, requests, dtype, seed=5, extra_pages=extra)
    is_bf16 = dtype == torch.bfloat16
    with probe.env_set(env):
        out, buf = run_beam(c, max_len=max_len, guarded=True)
        rows = run_rows(c, max_len=max_len)
    probe.RESULTS.clear()
    if max_len is None or max_len > int(c.seq.max()):
        B = len(requests)
        f64, E = orc.paged_decode_attn_np(c.q.view(B * W, Hq, D).float().numpy(), c.pool.float().numpy(), c.block_ids.numpy(),
                                          c.seq.numpy(), T, with_abs=True)
        ok, info = probe.budget_info(out, f64, E, is_bf16)
        probe.report(name + " [beam kernel vs float64, error budget]", ok, info)
    probe.report_bands(name, buf)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad
    tol = 2e-2 if is_bf16 else 1e-2
    np.testing.assert_allclose(out.float().cpu().numpy(), rows.float().cpu().numpy(), rtol=tol, atol=tol)


# ------------------------------------------------------------------------------------------------ 5. replay
def test_graph_replay_with_pdl_behind_the_kernel_that_writes_q_and_kv():
    """rope_append (writes q and the new token's K/V) then the beam attention, captured with PDL: every replay gives the bits
    of the two calls run eagerly without PDL on the same state, again after the lengths advance in place."""
    Hq, Hkv, T, D, W = 8, 2, 16, 128, 4
    # (three appended tokens stay inside every beam's last page)
    c = make_case(Hq, Hkv, T, D, W, [(128, [140, 129, 150, 170]), (64, [65, 100, 70, 85])], torch.float16, seed=6)
    R = c.seq.numel()
    g = torch.Generator().manual_seed(7)
    spec = rope.RopeSpec(dim=D, base=10000.0)
    qkv = torch.randn(R, (Hq + 2 * Hkv) * D, generator=g).half().to(DEV)
    pl = ops.convert_block_table(c.block_ids.to(DEV))
    shared, max_len = c.shared.to(DEV), int(c.seq.max()) + 4
    ws = ops.attn_workspace(R, Hq, Hkv, max_len, DEV)

    def two_calls(pool, seq, q, out):
        rope.rope_append(spec, qkv, pool, pl, seq, Hq, q_out=q)
        ops.paged_decode_attn_beam(q.view(-1, W, Hq, D), pool, pl, seq, shared, max_len, ws, out=out)
    bufs = lambda: (torch.empty(R, Hq * D, dtype=torch.float16, device=DEV), torch.empty(R // W, W, Hq * D, dtype=torch.float16,
                                                                                         device=DEV))
    pool_g, seq_g, (q_g, out_g) = c.pool.to(DEV), c.seq.to(DEV), bufs()
    pool_e, seq_e, (q_e, out_e) = c.pool.to(DEV), c.seq.to(DEV), bufs()
    try:
        ops.set_pdl(True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            two_calls(pool_g, seq_g, q_g, out_g)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            two_calls(pool_g, seq_g, q_g, out_g)
        ops.set_pdl(False)
        for step in range(3):
            out_g.zero_()
            graph.replay()
            two_calls(pool_e, seq_e, q_e, out_e)
            torch.cuda.synchronize()
            assert same_bits(out_g, out_e), f"replay {step} differs from the eager calls"
            assert same_bits(pool_g, pool_e)
            seq_g.add_(1)
            seq_e.add_(1)
    finally:
        ops.set_pdl(False)


# ------------------------------------------------------------------------------------------------ 7. the step
def _copy_state(dst: DecodeStep, src: DecodeStep):
    for name in ("ids", "seq_lens", "block_ids", "beam_cum", "hist", "hist_len"):
        getattr(dst, name).copy_(getattr(src, name))
    for Ld, Ls in zip(dst.layers, src.layers):
        Ld["kv"].copy_(Ls["kv"])
    if src.eos_id is not None:
        dst.hyp_state.copy_(src.hyp_state)
        dst.done.copy_(src.done)


@pytest.mark.parametrize("mode", ["eager", "graph+pdl"])
@pytest.mark.parametrize("quant,eos", [("int4", False), ("f16", True)], ids=["int4", "f16 eos"])
def test_beam_step_against_the_per_row_attention(quant, eos, mode):
    """DecodeStep(beam_width 4) over 9 steps with page crossings, next to the same step with the per-row attention started
    from the same state at every step: logits within the whole-step tolerance (and within it of the CPU oracle at the first
    step), K/V pools within tolerance, the same beams chosen wherever the candidates' scores are further apart than the logits
    can differ. At every step each request's page-table rows are equal over the pages shared_lens covers."""
    W, steps, T, B = 4, 9, TINY.tokens_per_block, 16
    cfg = dataclasses.replace(TINY, quant=quant, head_num=16, kv_head_num=8)     # 16 requests x 8 kv heads: the beam kernel's side
    kw = dict(keep_reference=True, ragged=True, seed=11, pdl="pdl" in mode, beam_width=W, max_new_tokens=12)
    if eos:
        kw.update(eos_id=7, length_penalty=0.8)
    new, old = DecodeStep(cfg, B, 200, DEV, **kw), PerRowBeamStep(cfg, B, 200, DEV, **kw)
    assert beam_rows_fit(new.Hq, new.Hkv, W, B)
    assert int(new.shared_lens.min()) >= 64, "the prompt is too short to share a 64-token tile"
    seq0 = new.seq_lens.cpu().long()
    assert ((seq0 + steps) // T > seq0 // T).any(), "no page crossing in this run"
    try:
        if "graph" in mode:
            new.capture()
            old.capture()
        clear = 0
        for t in range(steps):
            _copy_state(old, new)
            torch.cuda.synchronize()
            tbl, sh = new.block_ids.cpu().view(B, W, -1), new.shared_lens.cpu()
            for b in range(B):
                assert (tbl[b, :, :int(sh[b]) // T] == tbl[b, :1, :int(sh[b]) // T]).all(), f"step {t}: request {b}'s beams differ"
            if t == 0:
                state, kv_before = device_state(new), [step_bits(L["kv"]) for L in new.layers]
            for m in (new, old):
                m.replay() if "graph" in mode else m.run()
            torch.cuda.synchronize()
            got, ref = new.logits.float().cpu().numpy(), old.logits.float().cpu().numpy()
            if t == 0:
                check_logits(got, oracle_step(state, kv_before))
            err = check_logits(got, ref)
            for Ln, Lo in zip(new.layers, old.layers):
                torch.testing.assert_close(Ln["kv"].float(), Lo["kv"].float(), rtol=1e-2, atol=1e-2)
            # a candidate's score is log-softmax + cum: a logit error e moves it by at most 2e, so two candidates can only swap
            # when they are closer than 4e
            sel_n = {k: v.cpu().numpy() for k, v in new.beam_out.items()}
            sel_o = {k: v.cpu().numpy() for k, v in old.beam_out.items()}
            for b in range(B):
                sc = np.sort(sel_o["cand_score"][b].astype(np.float64))[::-1]
                if np.isfinite(sc).all() and (sc[:-1] - sc[1:]).min() > 4 * err + 1e-6:
                    clear += 1
                    for k in ("next_token", "next_parent"):
                        np.testing.assert_array_equal(sel_n[k][b], sel_o[k][b], err_msg=f"step {t} request {b}: {k}")
        assert clear > 0, "no request ever had candidates clear of the tolerance: the selections were not compared"
    finally:
        ops.set_pdl(False)


def test_the_step_takes_the_beam_kernel_only_when_the_rule_holds(monkeypatch):
    """group 2 x W 32 = 64 query rows fit a CTA and group 4 x W 32 = 128 do not; 2 requests x 8 kv heads are fewer pairs than
    the beam kernel was measured to win from. The steps outside the rule keep the per-row kernel. Counted on the two ops."""
    calls = {"beam": 0, "rows": 0}

    def counted(key, fn):
        def call(*a, **k):
            calls[key] += 1
            return fn(*a, **k)
        return call
    monkeypatch.setattr(ops, "paged_decode_attn_beam", counted("beam", ops.paged_decode_attn_beam))
    monkeypatch.setattr(ops, "paged_decode_attn", counted("rows", ops.paged_decode_attn))
    wide = dataclasses.replace(TINY_QWEN3, quant="int4", head_num=32, kv_head_num=8)       # group 4
    slim = dataclasses.replace(TINY_QWEN3, quant="int4", head_num=16, kv_head_num=8)       # group 2
    for cfg, B, W, fits in ((wide, 16, 8, True), (slim, 4, 32, False), (wide, 4, 32, False), (wide, 2, 8, False)):
        assert beam_rows_fit(cfg.head_num, cfg.kv_head_num, W, B) == fits
        model = DecodeStep(cfg, B, 120, DEV, beam_width=W, keep_reference=True, seed=3)
        state, kv_before = device_state(model), [step_bits(L["kv"]) for L in model.layers]
        calls.update(beam=0, rows=0)
        model.run()
        torch.cuda.synchronize()
        assert calls == ({"beam": cfg.layers, "rows": 0} if fits else {"beam": 0, "rows": cfg.layers}), (W, calls)
        check_logits(model.logits.float().cpu().numpy(), oracle_step(state, kv_before))


def test_beam_mode_counts_a_requests_shared_tokens_once():
    cfg = dataclasses.replace(TINY, quant="int4")
    W, B = 4, 2
    model = DecodeStep(cfg, B, 200, DEV, beam_width=W, max_new_tokens=12)
    per_token = 2.0 * model.Hkv * model.D * 2 * cfg.layers
    lens = (model.seq_lens_h.long() + 1).view(B, W)
    shared = model.shared_lens_h.long()
    assert model.algorithmic_bytes()["kv"] == per_token * float((shared + (lens - shared.view(B, 1)).sum(1)).sum())
    assert (shared == model.seq_lens_h.view(B, W)[:, 0] // cfg.tokens_per_block * cfg.tokens_per_block).all()
    greedy = DecodeStep(cfg, B, 200, DEV)
    assert greedy.algorithmic_bytes()["kv"] == per_token * float((greedy.seq_lens_h.long() + 1).sum())
