"""INT4 weights with quantisation group 64 / 32 (B200_FMT_INT4_G64 / _G32) and per-channel checkpoints on an H100: the blob
layout, the GEMM against the CPU oracle and the naive CUDA kernel, an exact probe of every group boundary, equivalence with
group 128, the fused SiLU*mul epilogue, PDL / CUDA-graph / decode-program replays, and checkpoints through the loader."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_INT4, B200_FMT_INT4_G32, B200_FMT_INT4_G64  # noqa: E402
from rtp_llm_b200.device import B200Impl  # noqa: E402
from rtp_llm_b200.linear import B200WeightOnlyLinear  # noqa: E402
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig  # noqa: E402
from tests import ckpt_util  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests import ref_kernels as refk  # noqa: E402
from tests.test_w4_groups import write_checkpoint  # noqa: E402

dev = torch.device("cuda")
FMT = {128: B200_FMT_INT4, 64: B200_FMT_INT4_G64, 32: B200_FMT_INT4_G32}


def bits(t):
    return t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def make_w4(K, N, group, seed=1):
    rng = np.random.default_rng(seed)
    qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
    s = (np.abs(rng.standard_normal((K // group, N))) * 0.01 + 1e-3).astype(np.float16)
    z = rng.integers(0, 16, (K // group, N))
    zs = ((8 - z).astype(np.float16) * s).astype(np.float16)
    return qp, s, zs


def to_dev(qp, s, zs, dtype):
    return torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dtype).to(dev), torch.from_numpy(zs).to(dtype).to(dev)


def expected_blob(qp, s, zs, group):
    """numpy restatement of the b200_pack_w4 layout (include/b200_decode_ops.h): per (128-feature tile, 128-k block), the
    nibbles u = q_s + 8 in wgmma fragment order, then group 128: 128 scales and 128 zero*scales; group 64 / 32: per group
    in k order, 128 {scale, zero*scale} pairs. s / zs are uint16 bits."""
    K, N = qp.shape[0], qp.shape[1] * 2
    nib = np.empty((K, N), np.uint32)
    nib[:, 0::2], nib[:, 1::2] = qp & 0xF, qp >> 4
    u = (nib + 8) & 0xF
    wi = np.arange(2048)
    vec = wi // 4
    R, lane, j = (vec // 32) % 8, vec % 32, (vec // 256) * 4 + wi % 4
    pos = np.arange(8)
    i, hi = pos & 3, pos >> 2
    row = 16 * R[:, None] + lane[:, None] // 4 + 8 * (i[None, :] & 1)                  # [2048, 8]
    kl = 16 * j[:, None] + 2 * (lane[:, None] & 3) + 8 * (i[None, :] >> 1) + hi[None, :]
    gpb = 128 // group
    out = []
    for tile in range((N + 127) // 128):
        n = tile * 128 + row
        ok = n < N
        cols = np.arange(tile * 128, tile * 128 + 128)
        cok = cols < N
        for kb in range(K // 128):
            vals = np.where(ok, u[kb * 128 + kl, np.minimum(n, N - 1)], 8)
            words = (vals << (4 * pos[None, :])).sum(axis=1).astype(np.uint32)
            parts = [words.view(np.uint8)]
            for g in range(gpb):
                sr = np.where(cok, s[kb * gpb + g, np.minimum(cols, N - 1)], 0).astype(np.uint16)
                zr = np.where(cok, zs[kb * gpb + g, np.minimum(cols, N - 1)], 0).astype(np.uint16)
                if gpb == 1:
                    parts += [sr.view(np.uint8), zr.view(np.uint8)]
                else:
                    parts.append(np.stack([sr, zr], 1).reshape(-1).view(np.uint8))
            out.append(np.concatenate(parts))
    return np.concatenate(out)


@pytest.mark.parametrize("group", [128, 64, 32])
def test_blob_bytes_match_the_layout(group):
    K, N = 256, 200
    qp, s, zs = make_w4(K, N, group)
    w = ops.pack_w4(*to_dev(qp, s, zs, torch.float16), group)
    torch.cuda.synchronize()
    assert w.fmt == FMT[group]
    got = w.data[:-256].cpu().numpy()
    exp = expected_blob(qp, s.view(np.uint16), zs.view(np.uint16), group)
    assert got.shape == exp.shape and np.array_equal(got, exp)
    again = ops.PackedWeight.from_tensor(w.data.clone())                       # the trailer carries the format
    assert (again.fmt, again.K, again.N) == (FMT[group], K, N)


def _gemm_vs_refs(group, B, K, N, dtype=torch.float16, bias=False, env=None):
    probe.RESULTS.clear()
    name = f"int4 g{group} B{B} K{K} N{N} {dtype} bias={bias} {env or ''}"
    with probe.env_set(env):
        rng = np.random.default_rng(2)
        x = torch.from_numpy(rng.standard_normal((B, K)).astype(np.float32)).to(dtype).to(dev)
        bias_t = torch.from_numpy(rng.standard_normal(N).astype(np.float32)).to(dtype).to(dev) if bias else None
        qp, s, zs = make_w4(K, N, group)
        qd, sd, zd = to_dev(qp, s, zs, dtype)
        w = ops.pack_w4(qd, sd, zd, group)
        ws = ops.gemm_workspace(B, [(K, N)], dev)
        buf, y = probe.guarded_empty((B, N), dtype)
        ops.wo_gemm(x, w, ws, bias=bias_t, out=y)
        ref = refk.ref_dequant_gemm(x, B200_FMT_INT4, qd, sd, zd, group, bias_t)
        torch.cuda.synchronize()
    is_bf16 = dtype == torch.bfloat16
    with probe.env_set(env):
        nsplit = probe.gemm_nsplit(K, N, False)
    probe.gemm_vs_f64(name, y, x, orc.dequant_exact("int4", qp, bits(sd), bits(zd), group, is_bf16), nsplit, is_bf16, bias=bias_t)
    # second opinions: the naive GPU kernel and the C oracle, at the reference's tolerance
    tol = 4e-2 if is_bf16 else 2e-2
    probe.report(name + " [kernel vs ref-kernel]", *probe.diff_info(y, ref.float().cpu().numpy(), tol, tol))
    exp = orc.dequant_gemm(bits(x), "int4", qp, scales=bits(sd), zeros_x_scales=bits(zd), group=group,
                           bias=bits(bias_t) if bias else None, is_bf16=is_bf16)
    probe.report(name + " [kernel vs oracle]", *probe.diff_info(y, orc.from_bits(exp, is_bf16), tol, tol))
    probe.report(name + " [semaphores reset]", int(ws[:16384].view(torch.int32).abs().sum().item()) == 0)
    probe.report_bands(name, buf)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad


GEMM_CASES = [
    (1, 1024, 256, torch.float16, True, None),
    (16, 1024, 256, torch.float16, False, None),
    (17, 1024, 384, torch.bfloat16, True, None),
    (64, 1024, 256, torch.float16, True, None),
    (65, 512, 256, torch.bfloat16, False, None),
    (128, 1024, 256, torch.float16, True, None),
    (128, 1024, 256, torch.bfloat16, False, None),
    (32, 1024, 256, torch.float16, False, {"B200_GEMM_SPLITK": 1}),
    (19, 1024, 384, torch.float16, True, {"B200_GEMM_SPLITK": 3}),
    (32, 2048, 256, torch.bfloat16, False, {"B200_GEMM_SPLITK": 8}),
    (17, 3200, 256, torch.float16, False, {"B200_GEMM_SPLITK": 1}),     # ring wrap: 25 blocks through the weight ring
    (33, 512, 136, torch.float16, True, None),                          # ragged last tile
]


@pytest.mark.parametrize("group", [64, 32])
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: f"B{c[0]}-K{c[1]}-N{c[2]}-{str(c[3])[6:]}-bias{int(c[4])}-{c[5] or ''}")
def test_gemm_matches_oracle_and_ref_kernel(group, case):
    B, K, N, dtype, bias, env = case
    _gemm_vs_refs(group, B, K, N, dtype, bias, env)


@pytest.mark.parametrize("group", [64, 32])
@pytest.mark.parametrize("shape", [(32, 4096, 6144), (32, 14336, 4096), (64, 4096, 28672)], ids=["qkv B32", "w2 B32", "w13 B64"])
def test_gemm_at_llama_shapes(group, shape):
    _gemm_vs_refs(group, *shape)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("group", [64, 32])
def test_group_boundaries_exact(group, dtype):
    """One-hot x on both sides of every group boundary of two k-blocks, a distinct power-of-two scale per group and zero*scale
    0: y = q_s * s exactly, so a scale taken from the neighbouring group shows up as a factor of two."""
    K, N = 256, 256
    ks = sorted({0, K - 1} | {b * group + d for b in range(1, K // group) for d in (-1, 0)})
    B = len(ks)
    rng = np.random.default_rng(4)
    qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
    G = K // group
    s = np.repeat((2.0 ** (np.arange(G) - G // 2))[:, None], N, 1).astype(np.float32)
    s *= np.where(np.arange(N) % 2, 1.0, 2.0)[None, :]                 # rows differ too (rows A and B of a fragment)
    x = torch.zeros(B, K, dtype=dtype)
    for b, k in enumerate(ks):
        x[b, k] = 1.0
    w = ops.pack_w4(torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dtype).to(dev), torch.zeros(G, N, dtype=dtype, device=dev),
                    group)
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    y = ops.wo_gemm(x.to(dev), w, ws).float().cpu().numpy()
    q = np.empty((K, N), np.int32)
    q[:, 0::2], q[:, 1::2] = qp & 0xF, qp >> 4
    q = np.where(q >= 8, q - 16, q)
    exp = np.stack([q[k] * s[k // group] for k in ks])
    assert np.array_equal(y, exp), np.argwhere(y != exp)[:8]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("group", [64, 32])
def test_shared_scales_equal_group_128(group, dtype):
    """Groups inside each 128-block sharing s and zero*s are a g128 weight: the outputs are the same bits at every batch pad."""
    K, N = 1024, 384
    qp, s, zs = make_w4(K, N, 128, seed=6)
    r = 128 // group
    q, s128, z128 = to_dev(qp, s, zs, dtype)
    w128 = ops.pack_w4(q, s128, z128)
    wg = ops.pack_w4(q, s128.repeat_interleave(r, 0).contiguous(), z128.repeat_interleave(r, 0).contiguous(), group)
    assert wg.fmt == FMT[group]
    for B in (16, 32, 64, 128):
        x = torch.randn(B, K, generator=torch.Generator().manual_seed(B)).to(dtype).to(dev)
        ws = ops.gemm_workspace(B, [(K, N)], dev)
        assert torch.equal(ops.wo_gemm(x, wg, ws).view(torch.int16), ops.wo_gemm(x, w128, ws).view(torch.int16)), B


@pytest.mark.parametrize("env", [None, {"B200_GEMM_SPLITK": 4}], ids=["direct", "cluster split"])
@pytest.mark.parametrize("group", [64, 32])
def test_fused_silu_mul(group, env):
    B, K, inter = 32, 1024, 128
    N = 2 * inter
    with probe.env_set(env):
        rng = np.random.default_rng(9)
        x = torch.from_numpy(rng.standard_normal((B, K)).astype(np.float32)).half().to(dev)
        qp, s, zs = make_w4(K, N, group)
        qd, sd, zd = to_dev(qp, s, zs, torch.float16)
        w = ops.pack_w4(ops.interleave_gate_up(qd, inter, packed_int4=True), ops.interleave_gate_up(sd, inter),
                        ops.interleave_gate_up(zd, inter), group)
        ws = ops.gemm_workspace(B, [(K, N)], dev)
        buf, y = probe.guarded_empty((B, inter), torch.float16)
        ops.wo_gemm(x, w, ws, silu_mul=True, out=y)
        torch.cuda.synchronize()
    gu = orc.dequant_gemm(bits(x), "int4", qp, scales=bits(sd), zeros_x_scales=bits(zd), group=group)
    probe.RESULTS.clear()
    with probe.env_set(env):
        nsplit = probe.gemm_nsplit(K, N, False)
    probe.silu_vs_f64("silu", y, x, orc.dequant_exact("int4", qp, bits(sd), bits(zd), group), nsplit, False)
    probe.report("silu", *probe.diff_info(y, orc.from_bits(orc.silu_and_mul(gu), False), 2e-2, 2e-2))
    probe.report_bands("silu", buf)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert not bad, bad


@pytest.mark.parametrize("group", [64, 32])
def test_pdl_and_graph_replay_are_bit_identical(group):
    B, K, N = 32, 4096, 4096                                           # 32 tiles: a cluster split along k
    qp, s, zs = make_w4(K, N, group)
    w = ops.pack_w4(*to_dev(qp, s, zs, torch.float16), group)
    x = torch.randn(B, K, generator=torch.Generator().manual_seed(1)).half().to(dev)
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    plain = ops.wo_gemm(x, w, ws).clone()
    pdl = ops.wo_gemm(x, w, ws, pdl=True).clone()
    y = torch.empty(B, N, dtype=torch.float16, device=dev)
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        ops.wo_gemm(x, w, ws, out=y)
    torch.cuda.current_stream().wait_stream(s_)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.wo_gemm(x, w, ws, out=y)
    y.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(pdl.view(torch.int16), plain.view(torch.int16))
    assert torch.equal(y.view(torch.int16), plain.view(torch.int16))


def test_decode_program_with_a_g64_gemm():
    """norm -> g64 GEMM -> norm recorded into a decode program: the norms become persistent-kernel ops, the GEMM its own
    cluster-kernel launch, whose output is the direct call's on the same input bit for bit. Replays repeat the same bits.
    (The persistent kernel's norm reduces in another order than the stand-alone norm kernel, so the norms are compared with
    the direct calls within a tolerance.)"""
    B, H = 8, 1024
    qp, s, zs = make_w4(H, H, 64)
    w = ops.pack_w4(*to_dev(qp, s, zs, torch.float16), 64)
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(B, H, generator=gen).half().to(dev)
    res0 = torch.randn(B, H, generator=gen).half().to(dev)
    g1, g2 = (torch.rand(H, generator=gen) + 0.5).half().to(dev), (torch.rand(H, generator=gen) + 0.5).half().to(dev)
    ws = ops.gemm_workspace(B, [(H, H)], dev)
    res, h, y, out = res0.clone(), torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)

    def calls():
        ops.add_rmsnorm(x, res, g1, 1e-5, out=h)
        ops.wo_gemm(h, w, ws, out=y)
        ops.add_rmsnorm(y, res, g2, 1e-5, out=out)
    calls()
    torch.cuda.synchronize()
    direct = (h.clone(), y.clone(), out.clone(), res.clone())
    prog = ops.Program()
    with prog.record():
        calls()
    assert prog.num_ops == 2                       # the norms run in the persistent kernel, the g64 GEMM as its own launch
    replays = []
    for _ in range(2):
        res.copy_(res0)
        for t in (h, y, out):
            t.zero_()
        prog.launch()
        torch.cuda.synchronize()
        replays.append(tuple(t.clone() for t in (h, y, out, res)))
    for a, b in zip(*replays):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    h_p, y_p = replays[0][0], replays[0][1]
    assert torch.equal(y_p.view(torch.int16), ops.wo_gemm(h_p, w, ws).view(torch.int16))
    for a, b in zip(replays[0], direct):
        assert (a.float() - b.float()).abs().max().item() <= 1e-2 * b.float().abs().max().item() + 1e-2


@pytest.mark.parametrize("group", [32, 64, -1])
@pytest.mark.parametrize("method", ["gptq", "awq"])
def test_layer_through_the_loader(tmp_path, method, group):
    rng = np.random.default_rng(7)
    path = str(tmp_path / "layer.safetensors")
    hidden, heads, kvh, D, inter, align = 512, 4, 2, 128, 640, 256
    names, dense = write_checkpoint(path, rng, method, group, hidden, heads, kvh, D, inter)
    ld = B200Loader(CheckpointReader(path), QuantConfig(method, group_size=group), device=dev, align_size=align)
    L = ld.layer(names, inter=inter)
    inter_p = 768
    assert L["qkv"].fmt == (FMT[group] if group > 0 else B200_FMT_INT4)
    x = torch.from_numpy(rng.standard_normal((9, hidden)).astype(np.float32)).half().to(dev)
    ws = ops.gemm_workspace(16, [(hidden, 2 * inter_p), (inter_p, hidden), (hidden, (heads + 2 * kvh) * D)], dev)

    def close(y, ref):
        ref = torch.from_numpy(ref).to(dev)
        assert (y.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 2e-2

    xf = x.float().cpu().numpy()
    close(ops.wo_gemm(x, L["qkv"], ws), xf @ np.concatenate([dense["q"], dense["k"], dense["v"]], 1))
    close(ops.wo_gemm(x, L["o"], ws), xf @ dense["o"])
    g, u = xf @ dense["gate"], xf @ dense["up"]
    act = ops.wo_gemm(x, L["w13"], ws, silu_mul=True)
    close(act[:, :inter], g / (1 + np.exp(-g)) * u)
    assert float(act[:, inter:].abs().max()) == 0.0
    a16 = act.float().cpu().numpy()
    close(ops.wo_gemm(act, L["w2"], ws), a16[:, :inter] @ dense["down"])


@pytest.mark.parametrize("method", ["gptq", "awq"])
def test_preprocess_hook_infers_group_64_and_survives_copies(method):
    """The reference loader calls preprocess_groupwise_weight_params with no group: the group comes from the scales' shape
    (a g64 weight used to be packed as g128, reading half of its scale rows)."""
    rng = np.random.default_rng(2)
    t, dense = ckpt_util.make_layer(rng, method, 512, 256, group=64)
    impl = B200Impl(dev)
    kernel, zs, scales = impl.preprocess_groupwise_weight_params(t["qweight"], t["qzeros"], t["scales"], "cuda", method == "gptq",
                                                                 method == "awq", 4)
    copy = {"w": kernel.clone()}["w"].cpu().to(dev).contiguous()
    lin = B200WeightOnlyLinear(copy, weight_scales=scales, quant_config=type("Cfg", (), {"get_method": lambda self: method})())
    assert lin.packed.fmt == B200_FMT_INT4_G64
    x = torch.from_numpy(rng.standard_normal((4, 512)).astype(np.float32)).half().to(dev)
    ref = torch.from_numpy(x.float().cpu().numpy() @ dense).to(dev)
    assert (lin(x).float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 2e-2
