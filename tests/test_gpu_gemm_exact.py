"""The weight-only GEMM (csrc/wo_gemm.cuh, and the GEMM op of the persistent kernel in csrc/decode_program.cuh) pinned to
exact answers on an H100. The contract, read from the kernels:

  * W' (T = fp16 / bf16): INT4 g128 / g64 / g32 and INT8 group-wise: round_T(q_s * s + zs), ONE rounding (hfma2);
    INT8 per-column: q_s, exact (the column scale is the epilogue's); FP16 / BF16 weights: W.
  * acc = sum_k x_k W'_k: exact products, accumulated in fp32 on the tensor cores; split-K partials stay fp32 and are merged
    in a fixed order (the cluster kernel's l2_merge, or the persistent kernel's split tiles, S a power of two <= 16).
  * y = round_T(fmaf(acc, cscale, bias)), cscale = 1 except for INT8 per-column.
  * SiLU*mul epilogue: __fdividef(g, 1 + __expf(-g)) * u on the fp32 g, u, rounded once.

Three checks, each on every kernel path (the cluster kernel unsplit and through l2_merge, the persistent kernel's whole and
split tiles, FP16 weights through shared memory, bias, INT8 column scales, SiLU*mul, PDL):
  * dequantisation probe: one-hot rows give y[b] = round_T(fmaf(W'[k_b], cscale, bias)) bit for bit, for every k;
  * accumulation probe: integer-valued data on a power-of-two grid whose every partial sum is exact in fp32 in any order,
    so y = round_T(sum) bit for bit at any K, split and batch; twice on one workspace, and under a CUDA graph with PDL behind
    the kernel that writes X;
  * realistic random data against the float64 reference within oracle.gemm_error_budget, with the correctly rounded
    fractions above oracle.GEMM_MIN_ROUNDED / GEMM_MIN_WITHIN_ONE.
Each case asserts the path it names: the split plan (b200_plan_gemm_split, which follows the B200_GEMM_SPLITK hook) or, for
the persistent kernel, that the program holds the GEMM as its one op."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import _lib, ops  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402

dev = torch.device("cuda")
GROUP = {"f16": 128, "int8": 128, "int4": 128, "int4g64": 64, "int4g32": 32, "int8g": 128}
DT = {"f16": torch.float16, "bf16": torch.bfloat16}


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def tdev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dtype).to(dev)


def plan(K, N):
    """(nsplit, k-blocks per split) the cluster kernel launches for a K x N weight (B200_GEMM_SPLITK included)."""
    ns, kbp = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().b200_plan_gemm_split(K, N, ctypes.byref(ns), ctypes.byref(kbp)), "b200_plan_gemm_split")
    return ns.value, kbp.value


# ---------------------------------------------------------------------------------------------- weights
def make_weight(fmt, K, N, is_bf16, rng, grid=False):
    """(host arrays for pack, W' float64 [K,N] as the kernel multiplies it, cscale float64 [N] or None).

    Realistic (grid=False): the suite's distributions -- INT4 scales 1e-3 + 0.01|N(0,1)| and zero points 0..15, so
    zs = round_T((8 - z) s) takes both signs and q_s = z - 8 leaves only the rounding residue of zs: W' values near zero,
    fp16 subnormals among them; INT8G the same at 8 bits; INT8 per-column scales near 3e-4; FP16 weights N(0, 0.05).
    Grid (grid=True): every W' an integer of at most 12 times a scale 2^-6 or 2^-5 that varies by group and column (INT8:
    the column scale), zeros integer multiples of the scale."""
    G = K // GROUP[fmt]
    f = 2.0 ** -6
    if fmt in ("int4", "int4g64", "int4g32", "int8g"):
        if grid:
            s = f * 2.0 ** rng.integers(0, 2, (G, N))
            zs = rng.integers(-4, 5, (G, N)) * s
            q = rng.integers(-8, 8, (K, N))
        else:
            s = orc.round_t(np.abs(rng.standard_normal((G, N))) * (0.01 if fmt != "int8g" else 2e-4) + (1e-3 if fmt != "int8g" else 3e-4),
                            is_bf16)
            hi = 16 if fmt != "int8g" else 256
            zs = orc.round_t((hi // 2 - rng.integers(0, hi, (G, N))) * s, is_bf16)
            q = rng.integers(-hi // 2, hi // 2, (K, N))
        if fmt == "int8g":
            raw = q.astype(np.int8)
            wd = orc.dequant_exact("int8g", raw, s, zs, GROUP[fmt], is_bf16)
        else:
            u = (q & 0xF).astype(np.uint8)
            raw = (u[:, 0::2] | (u[:, 1::2] << 4)).astype(np.uint8)
            wd = orc.dequant_exact("int4", raw, s, zs, GROUP[fmt], is_bf16)
        return (raw, s, zs), wd, None
    if fmt == "int8":
        q = rng.integers(-12, 13, (K, N)) if grid else rng.integers(-128, 128, (K, N))
        c = f * 2.0 ** rng.integers(0, 2, N) if grid else orc.round_t(np.abs(rng.standard_normal(N)) * 2e-4 + 3e-4, is_bf16)
        return (q.astype(np.int8), c), q.astype(np.float64), c
    if grid:
        w = rng.integers(-12, 13, (K, N)) * (f * 2.0 ** np.repeat(rng.integers(0, 2, (G, N)), 128, axis=0))
    else:
        w = orc.round_t(rng.standard_normal((K, N)) * 0.05, is_bf16)
    return (w,), w.astype(np.float64), None


def pack(fmt, host, dtype, silu_inter=None):
    """The packed weight; silu_inter: interleave gate / up columns for the fused SiLU*mul epilogue first."""
    il = (lambda t, **k: ops.interleave_gate_up(t, silu_inter, **k)) if silu_inter else (lambda t, **k: t)
    if fmt == "int8":
        q, c = host
        return ops.pack_w8(il(torch.from_numpy(q).to(dev)), il(tdev(c, dtype)))
    if fmt == "f16":
        return ops.pack_f16(il(tdev(host[0], dtype)))
    raw, s, zs = host
    sd, zd = il(tdev(s, dtype)), il(tdev(zs, dtype))
    if fmt == "int8g":
        return ops.pack_w8g(il(torch.from_numpy(raw).to(dev)), sd, zd)
    return ops.pack_w4(il(torch.from_numpy(raw).to(dev), packed_int4=True), sd, zd, GROUP[fmt])


def fma_f32(a, b, c):
    """fmaf(a, b, c) for T-valued float64 arrays: a * b is exact in float64, and a * b + c is too for the values these tests
    draw (asserted through the rounding error of the sum), so the one float32 rounding is the cast's."""
    p = a * b
    s = p + c
    bb = s - p
    assert np.all((p - (s - bb)) + (c - bb) == 0.0), "a*b + c is not exact in float64"
    return s.astype(np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------- a. dequantisation probe
def _dequant_probe(fmt, dt, N, program):
    """One-hot rows: y[b] = round_T(fmaf(W'[k_b], cscale, bias)) bit for bit, for every k of the weight (K 512), with a
    random bias on the odd columns. R rows per launch (128 for the cluster kernel, 64 for the persistent kernel, whose
    batch pad stops there), K / R launches; launch L covers half (or all) of k-block j = L // (128 / R), and row b of it
    takes the k at position (37 (b + R h) + 11 j) mod 128, h = L % (128 / R), so rows and k differ in every launch."""
    K = 512
    R = 64 if program else 128
    dtype, is_bf16 = DT[dt], dt == "bf16"
    rng = np.random.default_rng(sum(map(ord, fmt + dt)) * 1000 + N)
    host, wd, cscale = make_weight(fmt, K, N, is_bf16, rng)
    w = pack(fmt, host, dtype)
    bias = orc.round_t(rng.standard_normal(N), is_bf16)
    bias[::2] = 0.0                                                        # W' alone (subnormals included) reaches y here
    bias_t = tdev(bias, dtype)
    ws = ops.gemm_workspace(R, [(K, N)], dev)
    cs = np.ones(N) if cscale is None else cscale
    if not is_bf16 and fmt not in ("f16", "int8"):
        assert ((wd != 0) & (np.abs(wd) < 2.0 ** -14)).any(), "no fp16 subnormal W' drawn"
    x_d = torch.zeros(R, K, dtype=dtype, device=dev)
    buf, y = probe.guarded_empty((R, N), dtype)
    prog = None
    if program:
        prog = ops.Program()
        with prog.record():
            ops.wo_gemm(x_d, w, ws, bias=bias_t, out=y)
        assert prog.num_ops == 1, f"the GEMM is not the program's one persistent-kernel op (num_ops {prog.num_ops})"
    per = 128 // R
    for L in range(K // R):
        j, h = divmod(L, per)
        ks = 128 * j + (37 * (np.arange(R) + R * h) + 11 * j) % 128
        x = np.zeros((R, K))
        x[np.arange(R), ks] = 1.0
        x_d.copy_(tdev(x, dtype))
        y.view(torch.int16).fill_(probe.SENTINEL)
        if prog is not None:
            prog.launch()
        else:
            ops.wo_gemm(x_d, w, ws, bias=bias_t, out=y)
        torch.cuda.synchronize()
        exp = orc.f64_to_bits(fma_f32(wd[ks], cs[None, :], bias[None, :]), is_bf16)
        got = bits(y)
        bad = np.argwhere(got != exp)
        assert bad.size == 0, [(int(b), int(ks[b]), int(n), hex(got[b, n]), hex(exp[b, n])) for b, n in bad[:6]]
        probe.RESULTS.clear()
        probe.report_bands("dequant probe", buf)
        assert probe.RESULTS[0][1]


@pytest.mark.parametrize("N", [136, 200])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("fmt", list(GROUP))
def test_dequant_probe_exact(fmt, dt, N):
    """The cluster kernel, every weight format."""
    _dequant_probe(fmt, dt, N, program=False)


@pytest.mark.parametrize("N", [136, 200])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("fmt", ["int4", "int8"])
def test_dequant_probe_exact_persistent_kernel(fmt, dt, N):
    """The persistent kernel's GEMM op (a one-op decode program), for the formats it runs: INT4 g128 and INT8."""
    _dequant_probe(fmt, dt, N, program=True)


# ---------------------------------------------------------------------------------------------- the path matrix
# (name, fmt, B, K, N, dtype, env, path). path: ("cluster", nsplit) -- the plan the cluster kernel must launch (None: the
# default plan, whatever it is, reported); ("program",) -- the persistent kernel as a one-op decode program.
def C(ns):
    return ("cluster", ns)


P = ("program",)
S1 = {"B200_GEMM_SPLITK": 1}
CASES = [
    # cluster kernel, one CTA per tile (ring wrap: 25 k-blocks through every stage ring), every batch-pad edge
    ("unsplit ring wrap int4 B1", "int4", 1, 3200, 256, "f16", S1, C(1)),
    ("unsplit ring wrap int4 B16 bf16", "int4", 16, 3200, 256, "bf16", S1, C(1)),
    ("unsplit ring wrap int4g64 B17", "int4g64", 17, 3200, 256, "f16", S1, C(1)),
    ("unsplit ring wrap int4g32 B32 bf16", "int4g32", 32, 3200, 256, "bf16", S1, C(1)),
    ("unsplit ring wrap int8g B33", "int8g", 33, 3200, 256, "f16", S1, C(1)),
    ("unsplit ring wrap int8 B64 bf16", "int8", 64, 3200, 256, "bf16", S1, C(1)),
    ("unsplit ring wrap f16 B65", "f16", 65, 3200, 256, "f16", S1, C(1)),
    ("unsplit ring wrap f16 B128 bf16", "f16", 128, 3200, 256, "bf16", S1, C(1)),
    ("unsplit ring wrap int4 B128", "int4", 128, 3200, 256, "f16", S1, C(1)),
    # cluster kernel, split-K through l2_merge: even runs, runs of 3, 3, 2, and 8 splits clamped to the 3 k-blocks of K 384
    ("l2_merge 2 int4 B32", "int4", 32, 1024, 384, "f16", {"B200_GEMM_SPLITK": 2}, C(2)),
    ("l2_merge 3 int4 B19 bf16", "int4", 19, 1024, 384, "bf16", {"B200_GEMM_SPLITK": 3}, C(3)),
    ("l2_merge 4 int8 B65", "int8", 65, 1024, 384, "f16", {"B200_GEMM_SPLITK": 4}, C(4)),
    ("l2_merge 8 f16 B128 bf16", "f16", 128, 1024, 384, "bf16", {"B200_GEMM_SPLITK": 8}, C(8)),
    ("l2_merge 8 int8g B17", "int8g", 17, 1024, 384, "f16", {"B200_GEMM_SPLITK": 8}, C(8)),
    ("l2_merge 3 int4g32 B64 bf16", "int4g32", 64, 1024, 384, "bf16", {"B200_GEMM_SPLITK": 3}, C(3)),
    ("l2_merge 4 int4g64 B1", "int4g64", 1, 1024, 136, "f16", {"B200_GEMM_SPLITK": 4}, C(4)),
    ("l2_merge 8 clamped K384 int4 B33", "int4", 33, 384, 256, "f16", {"B200_GEMM_SPLITK": 8}, C(3)),
    ("l2_merge 8 clamped K384 f16 B16", "f16", 16, 384, 200, "f16", {"B200_GEMM_SPLITK": 8}, C(3)),
    # persistent kernel as a one-op program: split tiles, 16 contributors, whole tiles, several tiles per CTA, the
    # workspace-limited fallback (the workspace is sized for batch 16)
    ("persistent split int4 B32", "int4", 32, 1024, 256, "f16", None, P),
    ("persistent split int8 B17 bf16", "int8", 17, 1024, 384, "bf16", None, P),
    ("persistent 16 contributors int4 B32", "int4", 32, 2048, 128, "f16", None, P),
    ("persistent whole tiles int4 B1", "int4", 1, 128, 256, "f16", None, P),
    ("persistent whole tiles int8 B16 bf16", "int8", 16, 128, 256, "bf16", None, P),
    ("persistent several tiles per CTA int8 B8", "int8", 8, 256, 76800, "f16", None, P),
    ("persistent workspace for B16 int4 B40", "int4", 40, 1024, 256, "f16", None, P),
    ("persistent ragged N int4 B64 bf16", "int4", 64, 512, 200, "bf16", None, P),
    ("persistent Llama w2 int4 B32", "int4", 32, 14336, 4096, "f16", None, P),
    # the default plan at the real shapes: Llama-3-8B qkv / o / w13 / w2, the fp16 lm_head slice, the TP8 per-rank shapes
    ("Llama qkv int4 B32", "int4", 32, 4096, 6144, "f16", None, C(None)),
    ("Llama o int4 B32", "int4", 32, 4096, 4096, "f16", None, C(None)),
    ("Llama w13 int4 B64", "int4", 64, 4096, 28672, "f16", None, C(None)),
    ("Llama w2 int4 B32", "int4", 32, 14336, 4096, "f16", None, C(None)),
    ("Llama w2 int4 B32 bf16", "int4", 32, 14336, 4096, "bf16", None, C(None)),
    ("Llama w2 int4g32 B17", "int4g32", 17, 14336, 4096, "f16", None, C(None)),
    ("Llama qkv int8g B32", "int8g", 32, 4096, 6144, "f16", None, C(None)),
    ("Llama o int8 B32", "int8", 32, 4096, 4096, "f16", None, C(None)),
    ("lm_head slice f16 B32", "f16", 32, 4096, 16032, "f16", None, C(None)),
    ("TP8 qkv K4096 N768 int4 B32", "int4", 32, 4096, 768, "f16", None, C(None)),
    ("TP8 o K512 N4096 int4 B32", "int4", 32, 512, 4096, "f16", None, C(None)),
    ("TP8 w13 K4096 N3584 int4 B32", "int4", 32, 4096, 3584, "f16", None, C(None)),
    ("TP8 w2 K1792 N4096 int4 B32", "int4", 32, 1792, 4096, "f16", None, C(None)),
]
WS_BATCH = {"persistent workspace for B16 int4 B40": 16}


def check_path(case, prog=None):
    """Assert the case runs on the path it names; returns the nsplit its budget may assume (1 when not known: the loosest)."""
    name, fmt, B, K, N, dt, env, path = case
    if path[0] == "program":
        assert prog.num_ops == 1, f"{name}: the GEMM is not the program's one persistent-kernel op (num_ops {prog.num_ops})"
        return 1
    ns, kbp = plan(K, N)
    if path[1] is not None:
        assert ns == path[1], f"{name}: planned {ns} splits, the case is for {path[1]}"
    return ns


class Runner:
    """One case's GEMM on a fixed x buffer and workspace: eagerly, or recorded as a decode program (then launched)."""

    def __init__(self, case, w, dtype, bias_t=None, silu=False):
        name, fmt, B, K, N, dt, env, path = case
        self.x = torch.zeros(B, K, dtype=dtype, device=dev)
        self.buf, self.y = probe.guarded_empty((B, N // 2 if silu else N), dtype)
        self.ws = ops.gemm_workspace(WS_BATCH.get(name, B), [(K, N)], dev)
        self.call = lambda **k: ops.wo_gemm(self.x, w, self.ws, bias=bias_t, out=self.y, silu_mul=silu, **k)
        self.prog = None
        if path[0] == "program":
            self.prog = ops.Program()
            with self.prog.record():
                self.call()
        self.nsplit = check_path(case, self.prog)

    def __call__(self, x):
        self.x.copy_(x)
        self.y.view(torch.int16).fill_(probe.SENTINEL)
        if self.prog is not None:
            self.prog.launch()
        else:
            self.call()
        torch.cuda.synchronize()
        return bits(self.y)

    def clean(self):
        probe.RESULTS.clear()
        probe.report_bands("", self.buf)
        return probe.RESULTS[0][1] and int(self.ws[:24576].view(torch.int32).abs().sum().item()) == 0


def grid_x(B, K, rng):
    """x in {-1, 0, 1}: in every row, max(1, 48 // k-blocks) nonzeros in every k-block, at random positions and signs."""
    kb = K // 128
    per = max(1, 48 // kb)
    x = np.zeros((B, K))
    for b in range(B):
        pos = (np.arange(kb)[:, None] * 128 + np.stack([rng.choice(128, per, replace=False) for _ in range(kb)])).ravel()
        x[b, pos] = rng.choice([-1.0, 1.0], pos.size)
    return x


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_accumulation_probe_exact(case):
    """Integer-valued data on a power-of-two grid (finest step 2^-6): sum |x W'| + |bias| < 2^11 * 2^-6, so every partial
    sum, in any order, at any split and any tensor-core alignment, is exact in fp32, and y == round_T(sum) bit for bit. Run
    twice back to back on one workspace with different x (a partial left over from the first call shows), then captured in
    a CUDA graph behind the kernel that writes x (b200_permute_cols), with PDL."""
    name, fmt, B, K, N, dt, env, path = case
    dtype, is_bf16 = DT[dt], dt == "bf16"
    rng = np.random.default_rng(len(name) * 7919 + K)
    with probe.env_set(env):
        host, wd, cscale = make_weight(fmt, K, N, is_bf16, rng, grid=True)
        w = pack(fmt, host, dtype)
        bias = rng.integers(-64, 65, N) * 2.0 ** -6
        run = Runner(case, w, dtype, tdev(bias, dtype))
        for rep in range(2):
            x = grid_x(B, K, rng)
            ref, A = orc.gemm_np(x, wd, cscale, bias)
            assert A.max() < 2.0 ** 5, f"grid too coarse for exact sums: max sum |terms| {A.max()}"
            got = run(tdev(x, dtype))
            exp = orc.f64_to_bits(ref, is_bf16)
            bad = np.argwhere(got != exp)
            assert bad.size == 0, (f"call {rep}: {len(bad)} wrong", [(int(b), int(n), float(orc.from_bits(got[b:b + 1, n], is_bf16)[0]),
                                                                   ref[b, n]) for b, n in bad[:6]])
            assert run.clean(), f"call {rep}: guard band or workspace counters left dirty"
        if run.prog is not None:
            # a decode program is launched by Program.launch(), not by a stream of ops captured with the PDL flag, so the
            # graph + PDL run below is the cluster kernel's; the two eager calls above cover the persistent kernel
            return
        # graph + PDL: permute_cols writes x (and lets its dependents launch early); the GEMM must wait for it
        x_src = grid_x(B, K, rng)
        perm = rng.permutation(K)
        src, perm_t = tdev(x_src, dtype), torch.from_numpy(perm.astype(np.int32)).to(dev)
        x_in = torch.empty(B, K, dtype=dtype, device=dev)
        bias_t = tdev(bias, dtype)

        def step():
            ops.permute_cols(src, perm_t, out=x_in)
            ops.wo_gemm(x_in, w, run.ws, bias=bias_t, out=run.y, pdl=True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        run.y.view(torch.int16).fill_(probe.SENTINEL)
        x_in.zero_()
        g.replay()
        torch.cuda.synchronize()
        ref, _ = orc.gemm_np(x_src[:, perm], wd, cscale, bias)
        assert np.array_equal(bits(run.y), orc.f64_to_bits(ref, is_bf16)), "graph + PDL result differs"
        assert run.clean()


# ---------------------------------------------------------------------------------------------- c. float64 budget
def path_label(run, fmt):
    """The kernel path a case ran on, for the per-path figures of DESIGN section 4."""
    kind = "persistent" if run.prog is not None else ("cluster l2_merge" if run.nsplit > 1 else "cluster unsplit")
    return kind + (" f16-weights" if fmt == "f16" else "")


def budget_check(name, got, ref, A, K, nsplit, is_bf16, label=""):
    """Primary check of realistic data: every output within gemm_error_budget, and the correctly rounded fractions above
    their thresholds. Prints the worst err/budget and the fractions."""
    gv = orc.from_bits(got, is_bf16).astype(np.float64)
    ratio = np.abs(gv - ref) / orc.gemm_error_budget(ref, A, K, nsplit, is_bf16)
    ratio[np.isnan(ratio)] = np.inf
    eq, one = orc.gemm_rounded_fractions(got, ref, is_bf16)
    print(f"GEMMSTAT {name}: [{label} {'bf16' if is_bf16 else 'fp16'}] nsplit {nsplit} worst err/budget {ratio.max():.3f} "
          f"rounded {eq:.5f} within one step {one:.6f}")
    bad = np.argwhere(ratio > 1.0)
    assert bad.size == 0, [(int(b), int(n), gv[b, n], ref[b, n]) for b, n in bad[:6]]
    assert eq >= orc.GEMM_MIN_ROUNDED and one >= orc.GEMM_MIN_WITHIN_ONE, (eq, one)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_random_data_within_budget(case):
    """Realistic random weights and N(0, 1) activations (with a bias on the even-numbered cases) against the float64
    reference: the primary check of accuracy; the oracle and naive-kernel comparisons of test_gpu_parity are second
    opinions."""
    name, fmt, B, K, N, dt, env, path = case
    dtype, is_bf16 = DT[dt], dt == "bf16"
    rng = np.random.default_rng(len(name) * 104729 + N)
    with probe.env_set(env):
        host, wd, cscale = make_weight(fmt, K, N, is_bf16, rng)
        w = pack(fmt, host, dtype)
        bias = orc.round_t(rng.standard_normal(N), is_bf16) if CASES.index(case) % 2 == 0 else None
        run = Runner(case, w, dtype, None if bias is None else tdev(bias, dtype))
        x = orc.round_t(rng.standard_normal((B, K)), is_bf16)
        got = run(tdev(x, dtype))
        ref, A = orc.gemm_np(x, wd, cscale, bias)
        budget_check(name, got, ref, A, K, run.nsplit, is_bf16, path_label(run, fmt))
        assert run.clean()


SILU = [
    ("silu cluster unsplit int4 B7", "int4", 7, 256, 384, "f16", S1, C(1)),
    ("silu cluster unsplit int8 B33 bf16", "int8", 33, 1024, 256, "bf16", S1, C(1)),
    ("silu l2_merge 4 int4g64 B32", "int4g64", 32, 1024, 256, "f16", {"B200_GEMM_SPLITK": 4}, C(4)),
    ("silu l2_merge 3 f16 B17 bf16", "f16", 17, 1024, 384, "bf16", {"B200_GEMM_SPLITK": 3}, C(3)),
    ("silu l2_merge 8 int8g B65", "int8g", 65, 1024, 256, "f16", {"B200_GEMM_SPLITK": 8}, C(8)),
    ("silu persistent split int4 B32", "int4", 32, 1024, 256, "f16", None, P),
    ("silu persistent whole tiles int8 B7 bf16", "int8", 7, 128, 384, "bf16", None, P),
    ("silu Llama w13 int4 B64", "int4", 64, 4096, 28672, "f16", None, C(None)),
]


@pytest.mark.parametrize("case", SILU, ids=[c[0] for c in SILU])
def test_fused_silu_mul_within_budget(case):
    """The fused SiLU*mul epilogue on realistic data against silu(g) u of the float64 gate / up GEMMs, within
    oracle.silu_mul_budget (not bit-exact: __expf and __fdividef)."""
    name, fmt, B, K, N, dt, env, path = case
    dtype, is_bf16 = DT[dt], dt == "bf16"
    inter = N // 2
    rng = np.random.default_rng(len(name) * 31 + K)
    with probe.env_set(env):
        host, wd, cscale = make_weight(fmt, K, N, is_bf16, rng)
        w = pack(fmt, host, dtype, silu_inter=inter)
        run = Runner(case, w, dtype, silu=True)
        x = orc.round_t(rng.standard_normal((B, K)), is_bf16)
        got = orc.from_bits(run(tdev(x, dtype)), is_bf16).astype(np.float64)
        cg, cu = (None, None) if cscale is None else (cscale[:inter], cscale[inter:])
        g, Ag = orc.gemm_np(x, wd[:, :inter], cg)
        u, Au = orc.gemm_np(x, wd[:, inter:], cu)
        ref = orc.silu_mul_np(g, u)
        ratio = np.abs(got - ref) / orc.silu_mul_budget(g, Ag, u, Au, K, run.nsplit, is_bf16)
        ratio[np.isnan(ratio)] = np.inf
        print(f"GEMMSTAT {name}: [silu {path_label(run, fmt)} {'bf16' if is_bf16 else 'fp16'}] nsplit {run.nsplit} "
              f"worst err/budget {ratio.max():.3f}")
        assert ratio.max() <= 1.0, [(int(b), int(n), got[b, n], ref[b, n]) for b, n in np.argwhere(ratio > 1.0)[:6]]
        assert run.clean()
