"""The glue kernels pinned to float64 references (oracle.rmsnorm_np, rope_np, silu_mul_np) within their error budgets and
rounded-fraction thresholds, and the persistent kernel's glue ops (norm, rope + append, embedding, block-table conversion)
run as one-op decode programs, at the widths, positions and grid-stride edges where such kernels go wrong.

Each rope case writes into a pool of guard pages: every block-table entry points at one shared guard page except the
entry of each sequence's write slot, which has a page of its own, and the pool starts as a NaN sentinel. Everything outside
the one slot per (sequence, kv head) that the call writes must keep its bits."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import RopeConfig  # noqa: E402

dev = torch.device("cuda")
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
SENTINEL = {False: 0x7E01, True: 0x7FC1}                 # a quiet NaN with a payload no kernel computes


def is_bf16(dtype):
    return dtype == torch.bfloat16


def dev_t(v, dtype):
    """float64 T values -> a device tensor of dtype holding exactly those values."""
    return torch.from_numpy(orc.f64_to_bits(v, is_bf16(dtype)).view(np.int16)).view(dtype).to(dev)


def bits_of(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def report(what, got, ref, budget, frac_min, dtype, mask=None):
    """Asserts every output within its budget and the rounded fractions (over mask) above frac_min; prints the numbers."""
    bf = is_bf16(dtype)
    g = orc.from_bits(np.asarray(got, np.uint16), bf).astype(np.float64) if np.asarray(got).dtype == np.uint16 else got
    r = np.abs(g - ref) / budget
    bad = ~(r <= 1.0)
    m = np.ones(ref.shape, bool) if mask is None else mask
    gb = orc.f64_to_bits(g, bf)
    eq, one = orc.gemm_rounded_fractions(gb[m], ref[m], bf) if m.any() else (1.0, 1.0)
    worst = float(np.nanmax(np.where(np.isfinite(r), r, np.inf)))
    print(f"GLUE-STAT {what} {DT_IDS[bf]} worst {worst:.3f} rounded {eq:.5f} within-one {one:.6f} n {int(m.sum())}")
    assert not bad.any(), f"{what}: {int(bad.sum())} outputs outside the budget (worst err/budget {worst:.3g})"
    assert eq >= frac_min[0] and one >= frac_min[1], f"{what}: rounded / within one step {eq:.4f} / {one:.5f}"


NORM_FRAC = (orc.NORM_MIN_ROUNDED, orc.NORM_MIN_WITHIN_ONE)
SILU_FRAC = (orc.SILU_MIN_ROUNDED, orc.SILU_MIN_WITHIN_ONE)
ROPE_FRAC = (orc.ROPE_MIN_ROUNDED, orc.ROPE_MIN_WITHIN_ONE)


# ---------------------------------------------------------------------------------------------- RMSNorm
def norm_inputs(rows, hidden, dtype, seed, overflow=False):
    """x, residual, gamma as T values: N(0, 1) rows, every third row (from row 1) with an RMS near 1e-3, where eps matters.
    overflow: the first 8 entries of row 0 sum past fp16's largest value."""
    rng = np.random.default_rng(seed)
    bf = is_bf16(dtype)
    scale = np.where(np.arange(rows) % 3 == 1, 1e-3, 1.0)[:, None]
    x = orc.round_t(rng.standard_normal((rows, hidden)) * scale, bf)
    r = orc.round_t(rng.standard_normal((rows, hidden)) * scale, bf)
    if overflow:
        x[0, :8], r[0, :8] = 40000.0, 36000.0
    return x, r, orc.round_t(rng.uniform(0.5, 1.5, hidden), bf)


def standalone_threads(hidden):
    return 512 if hidden // 8 >= 512 else (256 if hidden // 8 >= 256 else 128)


NORM_CASES = [(8, 1, 1e-5), (1000, 33, 1e-6), (2048, 128, 1e-5), (3584, 7, 1e-6), (4096, 64, 1e-5), (5120, 16, 1e-6),
              (8192, 5, 1e-5), (12288, 3, 1e-6)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("with_res", [False, True], ids=["norm", "add_norm"])
@pytest.mark.parametrize("hidden,rows,eps", NORM_CASES)
def test_add_rmsnorm_within_budget(hidden, rows, eps, with_res, dtype):
    """b200_add_rmsnorm at every thread-count branch (128 / 256 / 512) up to its 12288 limit (a 48 KB staged row); fp16 rows
    with a residual also hold entries whose sum overflows: the stored residual is inf there and y stays finite."""
    overflow = with_res and not is_bf16(dtype)
    x, r, g = norm_inputs(rows, hidden, dtype, hidden + rows, overflow)
    ref, s, A = orc.rmsnorm_np(x, r if with_res else None, g, eps)
    res = dev_t(r, dtype) if with_res else None
    y = ops.add_rmsnorm(dev_t(x, dtype), res, dev_t(g, dtype), eps)
    torch.cuda.synchronize()
    if with_res:
        assert np.array_equal(bits_of(res), orc.f64_to_bits(s, is_bf16(dtype))), "stored residual is not round_T(x + r)"
        if overflow:
            assert torch.isinf(res[0, :8].float()).all() and torch.isfinite(y).all()
    budget = orc.norm_error_budget(ref, A, orc.norm_chain(hidden, standalone_threads(hidden)), is_bf16(dtype))
    report(f"add_rmsnorm standalone h{hidden}", bits_of(y), ref, budget, NORM_FRAC, dtype)


# ---------------------------------------------------------------------------------------------- SiLU*mul
SPECIAL_GATES = [20.0, -20.0, 88.0, -88.0, 100.0, -100.0]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("rows,inter", [(1, 2), (128, 14336), (128, 29696)])
def test_silu_and_mul_within_budget(rows, inter, dtype):
    """One pair, Llama-3-8B's 14336, and 29696 at 128 rows: past the grid cap, so the grid-stride loop runs. Gates at
    +-20 / +-88 / +-100, where __expf saturates, on the first rows."""
    rng = np.random.default_rng(inter)
    bf = is_bf16(dtype)
    gu = rng.standard_normal((rows, 2 * inter)) * 3
    sp = np.resize(np.array(SPECIAL_GATES), min(inter, 64))
    gu[0, :len(sp)] = sp
    gu = orc.round_t(gu, bf)
    y = ops.silu_and_mul(dev_t(gu, dtype))
    torch.cuda.synchronize()
    g, u = gu[:, :inter], gu[:, inter:]
    ref = orc.silu_mul_np(g, u)
    report(f"silu_and_mul standalone inter{inter}", bits_of(y), ref, orc.silu_mul_budget(g, 0.0, u, 0.0, 128, 1, bf), SILU_FRAC, dtype)


# ---------------------------------------------------------------------------------------------- RoPE + append
class GuardPool:
    """Block table [B, M] of the guard page 0 except each sequence's write-slot entry (page 1 + b), pool [1 + B, 2, Hkv, T, D]
    of NaN sentinels, and the expected pool after a call that writes K / V rows kv [B, 2, Hkv, D] (bits) at `slots`."""

    def __init__(self, slots, Hkv, T, D, dtype):
        self.slots = np.asarray(slots, np.int32)
        B = len(self.slots)
        M = int(self.slots.max()) // T + 1
        block_ids = np.zeros((B, M), np.int32)
        block_ids[np.arange(B), self.slots // T] = 1 + np.arange(B)
        self.page_list = torch.from_numpy(orc.convert_block_table(block_ids)).to(dev)
        self.seq = torch.from_numpy(self.slots).to(dev)
        self.T, self.shape = T, (1 + B, 2, Hkv, T, D)
        self.init = np.full(self.shape, SENTINEL[is_bf16(dtype)], np.uint16)
        self.pool = torch.from_numpy(self.init.view(np.int16)).view(dtype).to(dev)

    def fresh(self):
        return torch.from_numpy(self.init.view(np.int16)).view(self.pool.dtype).to(dev)

    def written(self, pool_bits):
        """The new K / V rows [B, 2, Hkv, D] the call wrote, after checking every other element kept its sentinel bits."""
        B = len(self.slots)
        keep = np.ones(self.shape, bool)
        keep[1 + np.arange(B), :, :, self.slots % self.T] = False
        assert np.array_equal(pool_bits[keep], self.init[keep]), \
            f"{int((pool_bits[keep] != self.init[keep]).sum())} pool elements outside the write slots changed"
        return pool_bits[1 + np.arange(B), :, :, self.slots % self.T]


def check_rope(what, q, pool_bits, gp, ref, R, dA, Hq, Hkv, D, dtype):
    """q_out and the pool of one rope call: guard pages and sentinels untouched, V a bit copy of the (bias-added) input,
    q and K within rope_error_budget and the rounded fractions over rope_fraction_mask."""
    bf = is_bf16(dtype)
    B = len(gp.slots)
    kv = gp.written(pool_bits)                                                   # [B, 2, Hkv, D]
    assert np.array_equal(kv[:, 1], orc.f64_to_bits(ref[:, Hq + Hkv:], bf)), "V is not a bit copy"
    got = np.concatenate([bits_of(q).reshape(B, Hq, D), kv[:, 0]], 1)
    ref, R, dA = ref[:, :Hq + Hkv], R[:, :Hq + Hkv], dA[:, :Hq + Hkv]
    report(what, got, ref, orc.rope_error_budget(ref, R, dA, bf), ROPE_FRAC, dtype, orc.rope_fraction_mask(ref, R, dA, bf))


def slot_positions(T, n_extra=0, seed=0):
    base = [0, 1, T - 1, T, 2 * T - 1, 2049, 8191, 32767, 131071]
    rng = np.random.default_rng(seed)
    return np.array(base + list(rng.integers(0, 131072, n_extra)), np.int32)


ROPE_CASES = [  # D, page, Hq, Hkv, base
    (64, 16, 8, 8, 10000.0), (128, 64, 32, 8, 500000.0), (256, 128, 16, 2, 1e6), (128, 16, 64, 8, 1e6),
    (64, 128, 32, 4, 500000.0), (256, 64, 8, 1, 10000.0), (128, 128, 16, 4, 1e6)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", ROPE_CASES, ids=[f"D{c[0]}-p{c[1]}-g{c[2] // c[3]}-b{c[4]:g}" for c in ROPE_CASES])
def test_rope_append_within_budget(case, dtype):
    D, T, Hq, Hkv, base = case
    pos = slot_positions(T)
    rng = np.random.default_rng(D + T)
    qkv = orc.round_t(rng.standard_normal((len(pos), (Hq + 2 * Hkv) * D)), is_bf16(dtype))
    gp = GuardPool(pos, Hkv, T, D, dtype)
    q = ops.rope_append(dev_t(qkv, dtype), gp.pool, gp.page_list, gp.seq, Hq, base)
    torch.cuda.synchronize()
    out, R, dA = orc.rope_np(qkv, Hq, Hkv, D, pos, base=base, is_bf16=is_bf16(dtype))
    check_rope(f"rope_append standalone D{D}", q, bits_of(gp.pool), gp, out, R, dA, Hq, Hkv, D, dtype)


BASE = dict(style=1, dim=128, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=2048, extrapolation_factor=1.0, mscale=1.0)
LONG = [0, 1, 15, 16, 2047, 2048, 2049, 8191, 8192, 32767, 65537, 131071]
EX_CASES = [  # name, cfg, options (pos: positions; slots: where K / V go when position_ids override them)
    ("base scale 4", dict(BASE, scale=4.0), dict(pos=LONG)),
    ("base 1e6", dict(BASE, base=1e6), dict(pos=LONG)),
    ("llama3.1", dict(BASE, style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192), dict(pos=LONG)),
    ("yarn", dict(BASE, style=5, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13), dict(pos=LONG)),
    ("dynamic ntk", dict(BASE, style=3, scale=2.0, max_pos=512), dict(pos=LONG)),
    ("qwen ntk steps", dict(BASE, style=4, max_pos=1024), dict(pos=[1022, 1023, 1024, 2046, 2047, 2048, 4094, 4095, 4096, 131071])),
    ("mrope", dict(BASE, style=7, scale=2.0), dict(pos=LONG)),
    ("cache boundary", dict(BASE), dict(cache=64, pos=[0, 5, 62, 63, 64, 65, 131071])),
    ("logn edge", dict(BASE, max_pos=16), dict(logn=True, pos=[0, 15, 16, 17, 18, 2049, 131071])),
    ("dim 64 + bias + position_ids", dict(BASE, dim=64, base=1e6),
     dict(bias=True, slots=[3, 17, 40, 300, 1000, 5], pid=[0, 2049, 0, 131071, 65535, 1])),
    ("no rope + bias", dict(BASE, style=0), dict(bias=True, pos=[0, 9, 131071])),
]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", EX_CASES, ids=[c[0] for c in EX_CASES])
def test_rope_append_ex_within_budget(case, dtype):
    """b200_rope_append_ex, every served style at long positions, and the contract's edges: the cos/sin cache at
    pos = cache_positions - 1 and cache_positions (a table of half the angle, so either side is told apart), logn at
    max_pos and max_pos + 1, Qwen's NTK step at seq_len = 2^k max_pos and +-1, bias, position_ids, rotary dim < head_dim."""
    name, cfg, opt = case
    bf = is_bf16(dtype)
    Hq, Hkv, D, T = 8, 2, 128, 16
    slots = np.asarray(opt.get("slots", opt.get("pos")), np.int32)
    pid = None if "pid" not in opt else np.asarray(opt["pid"], np.int32)
    pos = slots if pid is None else np.where(pid > 0, pid, slots)
    rng = np.random.default_rng(len(name))
    qkv = orc.round_t(rng.standard_normal((len(slots), (Hq + 2 * Hkv) * D)), bf)
    bias = orc.round_t(rng.standard_normal((Hq + 2 * Hkv) * D) * 0.1, bf) if opt.get("bias") else None
    cache = orc.rope_cache_base(cfg["dim"], cfg["base"], 2.0, opt["cache"] // 2) if opt.get("cache") else None
    gp = GuardPool(slots, Hkv, T, D, dtype)
    q = ops.rope_append_ex(dev_t(qkv, dtype), gp.pool, gp.page_list, gp.seq, Hq, RopeConfig(**cfg),
                           bias=None if bias is None else dev_t(bias, dtype),
                           position_ids=None if pid is None else torch.from_numpy(pid).to(dev),
                           cos_sin_cache=None if cache is None else torch.from_numpy(cache).to(dev), use_logn_attn=bool(opt.get("logn")))
    torch.cuda.synchronize()
    out, R, dA = orc.rope_np(qkv, Hq, Hkv, D, pos, cfg=cfg, bias=bias, cos_sin_cache=cache, use_logn=bool(opt.get("logn")), is_bf16=bf)
    check_rope(f"rope_append_ex '{name}'", q, bits_of(gp.pool), gp, out, R, dA, Hq, Hkv, D, dtype)


# ---------------------------------------------------------------------------------------------- QK-RMSNorm
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("with_bias", [False, True], ids=["no_bias", "bias"])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_qk_rmsnorm_within_budget(D, with_bias, dtype):
    """b200_qk_rmsnorm against the per-head float64 norm, the bias added before the one rounding to T; v heads untouched."""
    bf = is_bf16(dtype)
    rng = np.random.default_rng(D + with_bias)
    R, Hq, Hkv = 7, 8, 2
    scale = np.where(np.arange(R) % 3 == 1, 1e-3, 1.0)[:, None]
    x = orc.round_t(rng.standard_normal((R, (Hq + 2 * Hkv) * D)) * scale, bf)
    qg, kg = (orc.round_t(rng.uniform(0.5, 1.5, D), bf) for _ in range(2))
    qb, kb = (orc.round_t(0.1 * rng.standard_normal(D), bf) for _ in range(2)) if with_bias else (None, None)
    t = dev_t(x, dtype)
    ops.qk_rmsnorm(t, dev_t(qg, dtype), dev_t(kg, dtype), Hq, Hkv, D, 1e-6, None if qb is None else dev_t(qb, dtype),
                   None if kb is None else dev_t(kb, dtype))
    torch.cuda.synchronize()
    h = x.reshape(R, -1, D)
    yq, _, Aq = orc.rmsnorm_np(h[:, :Hq], None, qg, 1e-6, qb)
    yk, _, Ak = orc.rmsnorm_np(h[:, Hq:Hq + Hkv], None, kg, 1e-6, kb)
    ref, A = np.concatenate([yq, yk], 1), np.concatenate([Aq, Ak], 1)
    got = bits_of(t).reshape(R, -1, D)
    assert np.array_equal(got[:, Hq + Hkv:], orc.f64_to_bits(h[:, Hq + Hkv:], bf)), "v heads changed"
    report(f"qk_rmsnorm D{D}", got[:, :Hq + Hkv], ref, orc.norm_error_budget(ref, A, D // 32 + 5, bf), NORM_FRAC, dtype)


# ---------------------------------------------------------------------------------------------- persistent-kernel ops
def record(calls, ops_expected=1, launches_expected=1):
    prog = ops.Program()
    with prog.record():
        calls()
    assert prog.num_ops == ops_expected and prog.num_launches == launches_expected, \
        f"path: num_ops {prog.num_ops}, num_launches {prog.num_launches}"
    return prog


def launch_twice(prog, outs, reset=lambda: None):
    """Launches prog twice (reset() before each) and requires the same bits in every output; returns the first results."""
    got = []
    for _ in range(2):
        reset()
        for t in outs:
            t.zero_()
        prog.launch()
        torch.cuda.synchronize()
        got.append([t.clone() for t in outs])
    for a, b in zip(*got):
        assert torch.equal(a.view(torch.int16 if a.element_size() == 2 else torch.int32),
                           b.view(torch.int16 if b.element_size() == 2 else torch.int32)), "two launches gave different bits"
    return got[0]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("with_res", [False, True], ids=["norm", "add_norm"])
@pytest.mark.parametrize("rows", [1, 7, 64, 300])
@pytest.mark.parametrize("hidden", [512, 2048, 3584, 4096, 5120, 8192])
def test_seg_norm_program(hidden, rows, with_res, dtype):
    """The persistent kernel's norm up to its 8192 limit, at 300 rows (more than its 2 x 132 CTAs, so a CTA takes a second
    row): the stored residual has the stand-alone kernel's bits, y is within the budget of its own reduction order."""
    eps = 1e-5 if rows % 2 else 1e-6
    x, r, g = norm_inputs(rows, hidden, dtype, hidden * 7 + rows)
    ref, s, A = orc.rmsnorm_np(x, r if with_res else None, g, eps)
    xd, gd, y = dev_t(x, dtype), dev_t(g, dtype), torch.empty(rows, hidden, dtype=dtype, device=dev)
    r0 = dev_t(r, dtype)
    res = r0.clone() if with_res else None
    prog = record(lambda: ops.add_rmsnorm(xd, res, gd, eps, out=y))
    (y1,) = launch_twice(prog, [y], reset=(lambda: res.copy_(r0)) if with_res else (lambda: None))
    if with_res:
        res_standalone = r0.clone()
        ops.add_rmsnorm(xd, res_standalone, gd, eps)
        torch.cuda.synchronize()
        assert torch.equal(res.view(torch.int16), res_standalone.view(torch.int16)), "stored residual differs from the stand-alone kernel's"
    budget = orc.norm_error_budget(ref, A, orc.norm_chain(hidden, 256), is_bf16(dtype))
    report(f"seg_norm program h{hidden}", bits_of(y1), ref, budget, NORM_FRAC, dtype)


@pytest.mark.parametrize("tag", ["f16_512", "f16_4096", "bf16_512", "bf16_4096"])
def test_seg_norm_program_vs_flashinfer_outputs(golden_dir, tag):
    """The persistent kernel's norm against the outputs of flashinfer's kernels (the stand-alone kernel's bar: stored
    residual bit-exact, > 97 % of y bit-identical)."""
    gold = np.load(os.path.join(golden_dir, "flashinfer_glue_ops.npz"))
    dtype = torch.bfloat16 if tag.startswith("bf16") else torch.float16
    t = lambda k: torch.from_numpy(gold[f"{tag}_{k}"].copy()).view(dtype).to(dev)
    x, r0, w = t("x"), t("res"), t("w")
    y, y2, res = torch.empty_like(x), torch.empty_like(x), r0.clone()

    def calls():
        ops.add_rmsnorm(x, None, w, 1e-6, out=y)
        ops.add_rmsnorm(x, res, w, 1e-6, out=y2)
    prog = record(calls, ops_expected=2)
    launch_twice(prog, [y, y2], reset=lambda: res.copy_(r0))
    assert torch.equal(res, t("fused_res"))
    assert (y == t("rmsnorm")).float().mean().item() > 0.97
    assert (y2 == t("fused_y")).float().mean().item() > 0.97


def test_wide_norm_is_its_own_launch():
    """hidden 8200 is past the persistent kernel's norm: the program keeps the stand-alone kernel's launch and its bits."""
    rows, hidden = 5, 8200
    x, r, g = norm_inputs(rows, hidden, torch.float16, 1)
    xd, gd, r0 = dev_t(x, torch.float16), dev_t(g, torch.float16), dev_t(r, torch.float16)
    y, res = torch.empty_like(xd), r0.clone()
    prog = record(lambda: ops.add_rmsnorm(xd, res, gd, 1e-5, out=y), ops_expected=0, launches_expected=1)
    (y1,) = launch_twice(prog, [y], reset=lambda: res.copy_(r0))
    res_e = r0.clone()
    y_e = ops.add_rmsnorm(xd, res_e, gd, 1e-5)
    torch.cuda.synchronize()
    assert torch.equal(y1.view(torch.int16), y_e.view(torch.int16)) and torch.equal(res.view(torch.int16), res_e.view(torch.int16))


SEG_ROPE_CASES = [(64, 16, 8, 8, 10000.0, 9), (128, 64, 32, 8, 500000.0, 64), (256, 128, 16, 2, 1e6, 24), (128, 16, 64, 8, 1e6, 40),
                  (64, 128, 32, 4, 500000.0, 64)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", SEG_ROPE_CASES, ids=[f"D{c[0]}-p{c[1]}-g{c[2] // c[3]}-B{c[5]}" for c in SEG_ROPE_CASES])
def test_seg_rope_program_equals_rope_append(case, dtype):
    """The persistent kernel's rope op gives q_out and the whole guard-page pool with the bits of b200_rope_append."""
    D, T, Hq, Hkv, base, B = case
    pos = slot_positions(T, B - 9, seed=B)
    rng = np.random.default_rng(B + D)
    qkv = dev_t(orc.round_t(rng.standard_normal((B, (Hq + 2 * Hkv) * D)), is_bf16(dtype)), dtype)
    gp = GuardPool(pos, Hkv, T, D, dtype)
    q_ref = ops.rope_append(qkv, gp.pool, gp.page_list, gp.seq, Hq, base)
    torch.cuda.synchronize()
    pool_ref = gp.pool.clone()
    pool, q = gp.fresh(), torch.empty_like(q_ref)
    prog = record(lambda: ops.rope_append(qkv, pool, gp.page_list, gp.seq, Hq, base, q_out=q))
    launch_twice(prog, [q], reset=lambda: pool.copy_(gp.fresh()))
    assert torch.equal(q.view(torch.int16), q_ref.view(torch.int16)), "q_out differs from b200_rope_append"
    assert torch.equal(pool.view(torch.int16), pool_ref.view(torch.int16)), "the pool differs from b200_rope_append's"


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("rows", [1, 300])
@pytest.mark.parametrize("hidden", [8, 4096, 8192])
def test_seg_embed_program(hidden, rows, dtype):
    V = 1000
    rng = np.random.default_rng(hidden + rows)
    table = dev_t(orc.round_t(rng.standard_normal((V, hidden)), is_bf16(dtype)), dtype)
    ids_np = rng.integers(0, V, rows).astype(np.int32)
    ids_np[0] = V - 1
    ids_np[-1 if rows > 1 else 0] = 0 if rows > 1 else V - 1
    ids = torch.from_numpy(ids_np).to(dev)
    out = torch.empty(rows, hidden, dtype=dtype, device=dev)
    prog = record(lambda: ops.embedding(ids, table, out=out))
    (got,) = launch_twice(prog, [out])
    assert torch.equal(got.view(torch.int16), table[ids.long()].view(torch.int16))


def test_seg_block_table_program():
    """B 64 x M 2048 block ids: more than the persistent kernel's 2 x 132 CTAs x 256 threads, so its grid-stride loop runs."""
    B, M = 64, 2048
    ids_np = np.random.default_rng(0).integers(0, 1 << 20, (B, M)).astype(np.int32)
    ids = torch.from_numpy(ids_np).to(dev)
    out = torch.empty(B, 1, 2, M, dtype=torch.int32, device=dev)
    prog = record(lambda: ops.convert_block_table(ids, out=out))
    (got,) = launch_twice(prog, [out])
    assert np.array_equal(got.cpu().numpy(), orc.convert_block_table(ids_np))
