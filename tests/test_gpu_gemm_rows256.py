"""The weight-only GEMM at 129..256 rows (batch pad 256: one CTA per 128 features over all rows, each weight block staged and
dequantised once) pinned to the exact answers of test_gpu_gemm_exact on an H100: the dequantisation probe and the
accumulation probe bit for bit, realistic data within oracle.gemm_error_budget and the rounded fractions of DESIGN section 4,
unsplit and through l2_merge (2..8 splits, uneven runs included), bias, INT8 column scales, the fused SiLU*mul and act-order
weights, at the Llama-3-8B shapes too. Each case asserts its split plan and that the arrival counters are back at zero; PDL
hazard cases run the new instance behind a slow predecessor. The limits: 257 rows and the reduce-scatter GEMM above 128 rows
are refused."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import _lib, ops  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests import pdl_cases as pc  # noqa: E402
from tests import test_gpu_gemm_exact as ge  # noqa: E402
from tests import test_gpu_pdl_hazards as hz  # noqa: E402

dev = torch.device("cuda")
ROWS = [129, 130, 160, 192, 200, 255, 256]
FMTS = list(ge.GROUP)
SPLITS = [1, 2, 3, 4, 8]


def expected_nsplit(K, forced):
    """gemm_split under B200_GEMM_SPLITK=forced: runs of ceil(k_blocks / forced), the last one shorter."""
    kb = K // 128
    kbp = -(-kb // min(forced, kb, 8))
    return -(-kb // kbp)


def matrix():
    """Every format x dtype x row count; the split cycles through SPLITS so that each row count meets several, on K 1280
    (10 k-blocks: 3 splits run 4 + 4 + 2, 4 run 3 + 3 + 3 + 1, 8 run 2 x 5)."""
    cases, i = [], 0
    for fmt in FMTS:
        for dt in ("f16", "bf16"):
            for B in ROWS:
                S = SPLITS[i % len(SPLITS)]
                i += 1
                K, N = 1280, 256 if i % 2 else 200
                cases.append((f"{fmt} {dt} B{B} split {S} N{N}", fmt, B, K, N, dt, {"B200_GEMM_SPLITK": S}, ge.C(expected_nsplit(K, S))))
    return cases


MATRIX = matrix()
LLAMA = [   # the default plan at the Llama-3-8B shapes, 256 rows
    ("Llama qkv int4 B256", "int4", 256, 4096, 6144, "f16", None, ge.C(None)),
    ("Llama o int4 B256 bf16", "int4", 256, 4096, 4096, "bf16", None, ge.C(None)),
    ("Llama w2 int4 B256", "int4", 256, 14336, 4096, "f16", None, ge.C(None)),
    ("lm_head slice f16 B256", "f16", 256, 4096, 16032, "f16", None, ge.C(None)),
]


@pytest.mark.parametrize("B", [129, 200, 256])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("fmt", FMTS)
def test_dequant_probe_exact_rows256(fmt, dt, B):
    """One-hot rows, every k of a K 512 weight over ceil(512 / B) launches: y[b] = round_T(fmaf(W'[k_b], cscale, bias)) bit
    for bit, with a random bias on the odd columns."""
    K, N = 512, 200
    dtype, is_bf16 = ge.DT[dt], dt == "bf16"
    rng = np.random.default_rng(sum(map(ord, fmt + dt)) * 1000 + B)
    host, wd, cscale = ge.make_weight(fmt, K, N, is_bf16, rng)
    w = ge.pack(fmt, host, dtype)
    bias = orc.round_t(rng.standard_normal(N), is_bf16)
    bias[::2] = 0.0
    bias_t = ge.tdev(bias, dtype)
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    cs = np.ones(N) if cscale is None else cscale
    x_d = torch.zeros(B, K, dtype=dtype, device=dev)
    buf, y = probe.guarded_empty((B, N), dtype)
    order = np.concatenate([rng.permutation(K), rng.permutation(K)])
    for L in range(-(-K // B)):
        ks = order[L * B:(L + 1) * B]
        x = np.zeros((B, K))
        x[np.arange(B), ks] = 1.0
        x_d.copy_(ge.tdev(x, dtype))
        y.view(torch.int16).fill_(probe.SENTINEL)
        ops.wo_gemm(x_d, w, ws, bias=bias_t, out=y)
        torch.cuda.synchronize()
        exp = orc.f64_to_bits(ge.fma_f32(wd[ks], cs[None, :], bias[None, :]), is_bf16)
        bad = np.argwhere(ge.bits(y) != exp)
        assert bad.size == 0, [(int(b), int(ks[b]), int(n)) for b, n in bad[:6]]
        probe.RESULTS.clear()
        probe.report_bands("dequant probe", buf)
        assert probe.RESULTS[0][1]


@pytest.mark.parametrize("case", MATRIX + LLAMA, ids=[c[0] for c in MATRIX + LLAMA])
def test_accumulation_probe_exact_rows256(case):
    """test_gpu_gemm_exact's accumulation probe at 129..256 rows: bit for bit, twice on one workspace with new x, then in a
    CUDA graph with PDL behind the kernel that writes x; guard bands and arrival counters clean after every launch."""
    ge.test_accumulation_probe_exact(case)


@pytest.mark.parametrize("case", MATRIX + LLAMA, ids=[c[0] for c in MATRIX + LLAMA])
def test_random_data_within_budget_rows256(case):
    """Realistic weights and N(0, 1) activations (a bias on every other case) within the float64 budget, with the rounded
    fractions of DESIGN section 4."""
    name, fmt, B, K, N, dt, env, path = case
    dtype, is_bf16 = ge.DT[dt], dt == "bf16"
    rng = np.random.default_rng(len(name) * 104729 + N + B)
    with probe.env_set(env):
        host, wd, cscale = ge.make_weight(fmt, K, N, is_bf16, rng)
        w = ge.pack(fmt, host, dtype)
        bias = orc.round_t(rng.standard_normal(N), is_bf16) if B % 2 == 0 else None
        run = ge.Runner(case, w, dtype, None if bias is None else ge.tdev(bias, dtype))
        x = orc.round_t(rng.standard_normal((B, K)), is_bf16)
        got = run(ge.tdev(x, dtype))
        ref, A = orc.gemm_np(x, wd, cscale, bias)
        ge.budget_check(name, got, ref, A, K, run.nsplit, is_bf16, ge.path_label(run, fmt))
        assert run.clean()


SILU = [
    ("silu unsplit int4 B256", "int4", 256, 1024, 384, "f16", ge.S1, ge.C(1)),
    ("silu l2_merge 3 int8 B129 bf16", "int8", 129, 1280, 256, "bf16", {"B200_GEMM_SPLITK": 3}, ge.C(3)),
    ("silu l2_merge 8 int4g32 B200", "int4g32", 200, 1024, 256, "f16", {"B200_GEMM_SPLITK": 8}, ge.C(8)),
    ("silu unsplit f16 B200 bf16", "f16", 200, 1024, 384, "bf16", ge.S1, ge.C(1)),
    ("silu l2_merge 2 int8g B255", "int8g", 255, 1024, 256, "f16", {"B200_GEMM_SPLITK": 2}, ge.C(2)),
    ("silu Llama w13 int4 B256", "int4", 256, 4096, 28672, "f16", None, ge.C(None)),
]


@pytest.mark.parametrize("case", SILU, ids=[c[0] for c in SILU])
def test_fused_silu_mul_within_budget_rows256(case):
    """The fused SiLU*mul epilogue, staged in the idle activation ring at batch pad 256, within oracle.silu_mul_budget."""
    ge.test_fused_silu_mul_within_budget(case)


@pytest.mark.parametrize("fmt", ["int4", "int8g"])
@pytest.mark.parametrize("B", [160, 256])
def test_act_order_gather_and_gemm_rows256(fmt, B):
    """An act-order weight (rows sorted by a permutation): the gather + GEMM gives the bits of the plain GEMM on x[:, perm]."""
    K, N = 1024, 384
    g = torch.Generator().manual_seed(B)
    perm = torch.randperm(K, generator=g)
    x = torch.randn(B, K, generator=g).half().to(dev)
    w_perm = pc._weight(fmt, torch.float16, K, N, torch.Generator().manual_seed(7), perm=perm)
    w_plain = pc._weight(fmt, torch.float16, K, N, torch.Generator().manual_seed(7))
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    scratch = torch.empty(B, K, dtype=torch.float16, device=dev)
    got = ops.wo_gemm(x, w_perm, ws, x_perm=scratch)
    exp = ops.wo_gemm(x[:, perm.to(dev)].contiguous(), w_plain, ws)
    assert torch.equal(got.view(torch.int16), exp.view(torch.int16))
    assert int(ws[:24576].view(torch.int32).abs().sum()) == 0


def test_row_limits():
    """257 rows: refused, naming the limit; the reduce-scatter GEMM takes at most 128 rows."""
    lib = _lib.load()
    K, N = 1024, 256
    w = pc._weight("int4", torch.float16, K, N, torch.Generator().manual_seed(3))
    x = torch.zeros(257, K, dtype=torch.float16, device=dev)
    y = torch.empty(257, N, dtype=torch.float16, device=dev)
    ws = ops.gemm_workspace(256, [(K, N)], dev)
    rc = lib.b200_wo_gemm(w.fmt, 0, ctypes.c_void_p(x.data_ptr()), 257, K, N, ctypes.c_void_p(w.data.data_ptr()), None, None,
                          ctypes.c_void_p(y.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(), 0, None)
    assert rc == -1 and b"1..256" in lib.b200_last_error()
    regions = (ctypes.c_void_p * 2)(ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(ws.data_ptr()))
    rc = lib.b200_wo_gemm_rs(w.fmt, 0, ctypes.c_void_p(x.data_ptr()), 129, K, N, ctypes.c_void_p(w.data.data_ptr()), None, None,
                             ctypes.c_void_p(y.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(), 0, regions, 1 << 20, 0, 2,
                             None)
    assert rc == -1 and b"1..128" in lib.b200_last_error()


PDL = [
    pc.Case("gemm int4 g128 b256 unsplit", ("wo_gemm_kernel",), pc._gemm("int4", B=256), {pc.SPLITK: 1}),
    pc.Case("gemm int4 g128 b256 l2 merge", ("wo_gemm_kernel",), pc._gemm("int4", B=256), {pc.SPLITK: 4}),
    pc.Case("gemm f16 b200 silu_mul", ("wo_gemm_kernel",), pc._gemm("f16", B=200, silu=True), {pc.SPLITK: 2}),
]


@pytest.mark.parametrize("case", PDL, ids=[c.name for c in PDL])
def test_rows256_gemm_waits_for_its_grid_dependency(case):
    """The batch-pad-256 instance behind the slow-predecessor harness of test_gpu_pdl_hazards."""
    hz._run_case(case)
