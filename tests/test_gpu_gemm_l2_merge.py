"""Split-K merge of the plain weight-only GEMM through L2 (wo_gemm.cuh: l2_merge) on an H100: every forced split against the
CPU oracle and the naive CUDA kernel for every weight format, both activation types, bias and the fused SiLU*mul, batch pads
1..128; bit-stable CUDA-graph replays (the tile arrival counters reset themselves); two GEMMs sharing one workspace under
programmatic dependent launch; a workspace one byte short; sentinel bands around every output."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import _lib, ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8, B200_FMT_INT8G  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests.test_gpu_w4_groups import _gemm_vs_refs  # noqa: E402

dev = torch.device("cuda")
SPLITS = [2, 3, 4, 8]
# the workspace's counter area: [0, 16384) the persistent kernel's, [16384, 24576) the tile arrivals of l2_merge
SEM_BYTES = 24576


def _run(fn, *a, **k):
    probe.RESULTS.clear()
    fn(*a, **k)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad


def _counters_clear(ws):
    return int(ws[:SEM_BYTES].view(torch.int32).abs().sum().item()) == 0


# (B, dtype, bias): the batch pads 16 (B1, B17 is 32), 32, 64, 128
BATCHES = [(1, torch.float16, True), (17, torch.bfloat16, False), (32, torch.float16, False), (64, torch.bfloat16, True),
           (128, torch.float16, False)]


@pytest.mark.parametrize("fmt", [B200_FMT_F16, B200_FMT_INT8, B200_FMT_INT4, B200_FMT_INT8G], ids=["f16", "int8", "int4", "int8g"])
@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("batch", BATCHES, ids=[f"B{b[0]}" for b in BATCHES])
def test_forced_split_vs_oracle(fmt, split, batch):
    """K = 1024 (8 k-blocks): splits 2 / 4 / 8 take even runs, split 3 runs of 3, 3, 2. N = 384: three tiles."""
    B, dtype, bias = batch
    _run(probe.gemm_case, f"split{split} B{B}", fmt, B, 1024, 384, dtype=dtype, bias=bias, env={"B200_GEMM_SPLITK": split})


@pytest.mark.parametrize("group", [64, 32])
@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("batch", BATCHES, ids=[f"B{b[0]}" for b in BATCHES])
def test_forced_split_int4_groups_vs_oracle(group, split, batch):
    B, dtype, bias = batch
    _gemm_vs_refs(group, B, 1024, 384, dtype=dtype, bias=bias, env={"B200_GEMM_SPLITK": split})


@pytest.mark.parametrize("fmt", [B200_FMT_F16, B200_FMT_INT8, B200_FMT_INT4, B200_FMT_INT8G], ids=["f16", "int8", "int4", "int8g"])
@pytest.mark.parametrize("split", SPLITS)
def test_forced_split_fused_silu_mul_vs_oracle(fmt, split):
    _run(probe.gemm_silu_case, f"silu split{split}", fmt, 32, 1024, 128, env={"B200_GEMM_SPLITK": split})
    _run(probe.gemm_silu_case, f"silu split{split} B17", fmt, 17, 1024, 192, env={"B200_GEMM_SPLITK": split})


@pytest.mark.parametrize("split", SPLITS)
def test_forced_split_fused_silu_mul_bf16_matches_unsplit(split):
    """bf16 activations through the fused SiLU*mul: the split result against the unsplit one (which the oracle tests
    check), within the rounding of the reordered fp32 sums."""
    B, K, inter = 17, 1024, 192
    w = _w4(K, 2 * inter, 4, torch.bfloat16)
    x = torch.randn(B, K, generator=torch.Generator(device=dev).manual_seed(5), device=dev).bfloat16()
    out = {}
    for s in (1, split):
        with probe.env_set({"B200_GEMM_SPLITK": s}):
            ws = ops.gemm_workspace(B, [(K, 2 * inter)], dev)
            buf, y = probe.guarded_empty((B, inter), torch.bfloat16)
            ops.wo_gemm(x, w, ws, out=y, silu_mul=True)
            torch.cuda.synchronize()
            assert _counters_clear(ws)
            probe.RESULTS.clear()
            probe.report_bands(f"silu bf16 split{s}", buf)
            assert probe.RESULTS[0][1]
            out[s] = y.float()
    torch.testing.assert_close(out[split], out[1], rtol=4e-2, atol=4e-2 * float(out[1].abs().mean()))


def _w4(K, N, seed, dtype=torch.float16):
    """INT4 group-128 weight with scales in the activation type."""
    qp, s, zs = probe.make_w4(K, N, seed=seed)
    return ops.pack_w4(torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dev).to(dtype), torch.from_numpy(zs).to(dev).to(dtype))


def _plan(K, N):
    """The split-K the library plans for a K x N weight."""
    ns, kbp = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().b200_plan_gemm_split(K, N, ctypes.byref(ns), ctypes.byref(kbp)), "b200_plan_gemm_split")
    return ns.value


def test_graph_replays_are_bit_stable():
    """Llama-3-8B o projection at batch 32 (planned split 8): 50 replays of a captured GEMM give the eager result bit for
    bit, which needs every tile's arrival counter back at zero after each launch."""
    K, N, B = 4096, 4096, 32
    assert _plan(K, N) > 1
    w = _w4(K, N, 1)
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    x = torch.randn(B, K, generator=torch.Generator(device=dev).manual_seed(0), device=dev).half()
    ref = ops.wo_gemm(x, w, ws).clone()
    torch.cuda.synchronize()
    assert _counters_clear(ws)
    y = torch.empty_like(ref)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.wo_gemm(x, w, ws, out=y, pdl=True)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.wo_gemm(x, w, ws, out=y, pdl=True)
    for i in range(50):
        y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int16), ref.view(torch.int16)), f"replay {i} differs"
    assert _counters_clear(ws)


def test_two_gemms_share_a_workspace_under_pdl():
    """o then w2 shapes chained (the second reads the first's output) in one graph, both split-K, both launched with PDL on
    one workspace: the second may start while the first drains, yet must not touch the workspace before the first is done.
    Bit-equal to the same GEMMs run one at a time with a synchronise between them."""
    B, K1, N1, N2 = 32, 4096, 4096, 2048
    assert _plan(K1, N1) > 1 and _plan(N1, N2) > 1
    w1, w2 = _w4(K1, N1, 1), _w4(N1, N2, 2)
    ws = ops.gemm_workspace(B, [(K1, N1), (N1, N2)], dev)
    x = torch.randn(B, K1, generator=torch.Generator(device=dev).manual_seed(3), device=dev).half()
    y1_ref = ops.wo_gemm(x, w1, ws).clone()
    torch.cuda.synchronize()
    y2_ref = ops.wo_gemm(y1_ref, w2, ws).clone()
    torch.cuda.synchronize()
    y1 = torch.empty_like(y1_ref)
    y2 = torch.empty_like(y2_ref)

    def step():
        ops.wo_gemm(x, w1, ws, out=y1, pdl=True)
        ops.wo_gemm(y1, w2, ws, out=y2, pdl=True)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(20):
        y1.zero_()
        y2.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y1.view(torch.int16), y1_ref.view(torch.int16))
        assert torch.equal(y2.view(torch.int16), y2_ref.view(torch.int16))
    assert _counters_clear(ws)


def test_workspace_one_byte_short_is_an_argument_error():
    K, N, B = 4096, 4096, 32
    assert _plan(K, N) > 1
    w = _w4(K, N, 1)
    need = int(_lib.load().b200_wo_gemm_workspace_bytes(B, N, K))
    x = torch.zeros(B, K, device=dev).half()
    ops.wo_gemm(x, w, torch.zeros(need, dtype=torch.uint8, device=dev))
    torch.cuda.synchronize()
    with pytest.raises(_lib.B200Error, match="too small for .* split-K partials"):
        ops.wo_gemm(x, w, torch.zeros(need - 1, dtype=torch.uint8, device=dev))


def test_workspace_covers_every_forced_split():
    """The size comes from the same plan as the launch, test hook included: each forced split fits the workspace it sizes."""
    B, K, N = 128, 1024, 384
    for split in SPLITS:
        with probe.env_set({"B200_GEMM_SPLITK": split}):
            need = int(_lib.load().b200_wo_gemm_workspace_bytes(B, N, K))
            assert need >= SEM_BYTES + 3 * split * 128 * 128 * 4
