"""GPTQ act-order (desc_act) weights on an H100: the column gather b200_permute_cols (eager, CUDA graph + PDL, decode program),
the GEMM of a weight that carries its row order, the loader on act-order checkpoints (qkv, o, fused SiLU w13 and the w2 order
folded into w13), blob copies, and DecodeStep(act_order=True) against the step oracle, also with q_len > 1 and Llama-3.1 rope."""
import dataclasses
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200Error  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep  # noqa: E402
from rtp_llm_b200.device import B200Impl  # noqa: E402
from rtp_llm_b200.linear import B200WeightOnlyLinear  # noqa: E402
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig  # noqa: E402
from tests import act_order_ckpt  # noqa: E402
from tests.step_oracle import TINY31, check_step  # noqa: E402

dev = torch.device("cuda")
DT = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def rand_perm(K, seed):
    return torch.randperm(K, generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------------------------------------- the gather kernel
@pytest.mark.parametrize("K", [128, 4096, 14336, 29696])
@pytest.mark.parametrize("rows", [1, 9, 32, 128])
@pytest.mark.parametrize("dtype", DT, ids=DT_IDS)
def test_permute_cols_equals_index_select(dtype, rows, K):
    x = torch.randn(rows, K, generator=torch.Generator().manual_seed(rows * 7 + K)).to(dtype).to(dev)
    perm = rand_perm(K, K).to(torch.int32).to(dev)
    y = torch.full_like(x, float("nan"))
    ops.permute_cols(x, perm, out=y)
    assert same_bits(y, x.index_select(1, perm.long()))


@pytest.mark.parametrize("dtype", DT, ids=DT_IDS)
def test_permute_cols_under_graph_with_pdl_and_in_a_program(dtype):
    """norm -> gather -> norm chains: under a CUDA graph with PDL (the gather waits for the norm that writes its input, and the
    norm after it for the gather), and recorded into a decode program (the norms run in the persistent kernel, the gather as
    its own launch). The gather is a bit copy of what the norm wrote."""
    rows, K = 32, 4096
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(rows, K, generator=gen).to(dtype).to(dev)
    g1 = (torch.rand(K, generator=gen) + 0.5).to(dtype).to(dev)
    perm = rand_perm(K, 1).to(torch.int32).to(dev)
    h, hp, out = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)

    def calls():
        ops.add_rmsnorm(x, None, g1, 1e-5, out=h)
        ops.permute_cols(h, perm, out=hp)
        ops.add_rmsnorm(hp, None, g1, 1e-5, out=out)

    try:
        ops.set_pdl(True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            calls()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            calls()
        for _ in range(3):
            hp.zero_()
            h.zero_()
            graph.replay()
            torch.cuda.synchronize()
            assert same_bits(hp, h.index_select(1, perm.long()))
    finally:
        ops.set_pdl(False)
    prog = ops.Program()
    with prog.record():
        calls()
    assert prog.num_launches == 3 and prog.num_ops == 2          # norm | gather | norm
    hp.zero_()
    prog.launch()
    torch.cuda.synchronize()
    assert same_bits(hp, h.index_select(1, perm.long()))


# ---------------------------------------------------------------------------------------------- GEMM with a row order
def _weight(bits, group, K, N, dtype, seed):
    rng = np.random.default_rng(seed)
    if bits == 4:
        q = torch.from_numpy(rng.integers(0, 256, (K, N // 2)).astype(np.uint8))
        s = torch.from_numpy((np.abs(rng.standard_normal((K // group, N))) * 0.01 + 1e-3).astype(np.float32)).to(dtype)
        zs = (torch.from_numpy(8 - rng.integers(0, 16, (K // group, N))).to(dtype) * s).to(dtype)
        b = q.numpy().astype(np.int32)
        qs = np.empty((K, N), np.int32)
        qs[:, 0::2], qs[:, 1::2] = b & 0xF, b >> 4
        qs = np.where(qs >= 8, qs - 16, qs)
    else:
        q = torch.from_numpy(rng.integers(-128, 128, (K, N)).astype(np.int8))
        s = torch.from_numpy((np.abs(rng.standard_normal((K // group, N))) * 6e-4 + 6e-5).astype(np.float32)).to(dtype)
        zs = (torch.from_numpy(128 - rng.integers(0, 256, (K // group, N))).to(dtype) * s).to(dtype)
        qs = q.numpy().astype(np.int32)
    dense_sorted = qs * np.repeat(s.float().numpy(), group, 0) + np.repeat(zs.float().numpy(), group, 0)
    return q.to(dev), s.to(dev), zs.to(dev), dense_sorted


def _pack(bits, q, s, zs, group, perm=None):
    return ops.pack_w4(q, s, zs, group, perm=perm) if bits == 4 else ops.pack_w8g(q, s, zs, group, perm=perm)


def _close(y, ref, tol):
    ref = torch.as_tensor(ref, dtype=torch.float32, device=y.device)
    err = (y.float() - ref).abs().max().item()
    assert err <= tol * ref.abs().max().item() + tol, (err, ref.abs().max().item())


@pytest.mark.parametrize("dtype", DT, ids=DT_IDS)
@pytest.mark.parametrize("bits,group", [(4, 128), (4, 64), (4, 32), (8, 128)], ids=["int4-g128", "int4-g64", "int4-g32", "int8g-g128"])
def test_wo_gemm_gathers_x_for_a_weight_with_a_row_order(bits, group, dtype):
    B, K, N = 9, 1024, 384
    q, s, zs, dense_sorted = _weight(bits, group, K, N, dtype, seed=group + bits)
    perm = rand_perm(K, 3)
    w_perm, w_plain = _pack(bits, q, s, zs, group, perm), _pack(bits, q, s, zs, group)
    assert w_plain.perm is None and torch.equal(w_perm.perm.cpu().long(), perm)
    assert torch.equal(w_perm.data[:w_plain.data.numel() - 256], w_plain.data[:-256])    # same blob bytes, then the perm
    x = torch.randn(B, K, generator=torch.Generator().manual_seed(2)).to(dtype).to(dev)
    ws = ops.gemm_workspace(16, [(K, N)], dev)
    buf = torch.empty(16, K, dtype=dtype, device=dev)
    y = ops.wo_gemm(x, w_perm, ws, x_perm=buf)
    assert same_bits(y, ops.wo_gemm(x[:, perm.to(dev)].contiguous(), w_plain, ws))
    # the dense weight the act-order checkpoint means: its row perm[j] is sorted row j
    dense = np.empty_like(dense_sorted)
    dense[perm.numpy()] = dense_sorted
    _close(y, x.float().cpu().numpy() @ dense, 2e-2 if bits == 4 else 1e-2)
    with pytest.raises(B200Error, match="x_perm"):
        ops.wo_gemm(x, w_perm, ws)
    with pytest.raises(B200Error, match="x_perm must be"):
        ops.wo_gemm(x, w_perm, ws, x_perm=buf[:4])


def test_blob_copies_keep_the_row_order():
    K, N, group = 1024, 256, 128
    q, s, zs, _ = _weight(4, group, K, N, torch.float16, seed=4)
    perm = rand_perm(K, 8)
    w = ops.pack_w4(q, s, zs, group, perm=perm)
    f = io.BytesIO()
    torch.save({"kernel": w.data}, f)
    f.seek(0)
    copies = [w.data.clone().cpu().to(dev), torch.load(f)["kernel"].to(dev)]
    cfg = type("Cfg", (), {"get_method": lambda self: "gptq"})()
    x = torch.randn(5, K, generator=torch.Generator().manual_seed(1)).half().to(dev)
    ref = B200WeightOnlyLinear(w.data, weight_scales=s, quant_config=cfg)(x)
    assert same_bits(ref, ops.wo_gemm(x[:, perm.to(dev)].contiguous(), ops.pack_w4(q, s, zs, group), ops.gemm_workspace(16, [(K, N)], dev)))
    for c in copies:
        again = ops.PackedWeight.from_tensor(c)
        assert torch.equal(again.perm.cpu().long(), perm)
        assert same_bits(B200WeightOnlyLinear(c, weight_scales=s, quant_config=cfg)(x), ref)


# ---------------------------------------------------------------------------------------------- checkpoints
@pytest.mark.parametrize("bits", [4, 8])
def test_trivial_g_idx_gives_the_same_blob_and_act_order_the_dense_weight(bits):
    rng = np.random.default_rng(6)
    K, N, group = 512, 256, 128
    impl = B200Impl(dev)
    trivial = (np.arange(K) // group).astype(np.int32)
    t, *_ = act_order_ckpt.make_act_order_layer(rng, K, N, trivial, group, bits)
    plain, _, _ = impl.preprocess_groupwise_weight_params(t["qweight"], t["qzeros"], t["scales"], "cuda", True, False, bits)
    with_gidx, _, _ = impl.preprocess_groupwise_weight_params(t["qweight"], t["qzeros"], t["scales"], "cuda", True, False, bits,
                                                              g_idx=t["g_idx"])
    torch.cuda.synchronize()
    assert torch.equal(plain, with_gidx)
    g_idx = act_order_ckpt.act_order_g_idx(rng, K, group)
    t, dense, *_ = act_order_ckpt.make_act_order_layer(rng, K, N, g_idx, group, bits)
    kernel, _, scales = impl.preprocess_groupwise_weight_params(t["qweight"], t["qzeros"], t["scales"], "cuda", True, False, bits,
                                                                g_idx=t["g_idx"])
    lin = B200WeightOnlyLinear(kernel.clone(), weight_scales=scales, quant_config=type("Cfg", (), {"get_method": lambda self: "gptq"})())
    assert lin.packed.perm is not None
    x = torch.randn(7, K, generator=torch.Generator().manual_seed(3)).half().to(dev)
    _close(lin(x), x.float().cpu().numpy() @ dense, 2e-2 if bits == 4 else 1e-2)


@pytest.mark.parametrize("bits,group", [(4, 128), (4, 64), (4, 32), (8, 128)], ids=["int4-g128", "int4-g64", "int4-g32", "int8g-g128"])
def test_layer_through_the_loader(tmp_path, bits, group):
    rng = np.random.default_rng(7)
    path = str(tmp_path / "layer.safetensors")
    hidden, heads, kvh, D, inter, align, inter_p = 512, 4, 2, 128, 640, 256, 768
    names, dense, gi = act_order_ckpt.write_act_order_checkpoint(path, rng, hidden, heads, kvh, D, inter, group, bits)
    ld = B200Loader(CheckpointReader(path), QuantConfig("gptq", bits=bits, group_size=group), device=dev, align_size=align)
    L = ld.layer(names, inter=inter)
    assert L["w13_fused_silu"] and L["qkv"].perm is not None and L["o"].perm is not None and L["w13"].perm is not None
    assert L["w2"].perm is None                                         # folded into w13
    p2 = ld.act_order([names["down"]])
    tol = 2e-2 if bits == 4 else 1e-2
    x = torch.from_numpy(rng.standard_normal((9, hidden)).astype(np.float32)).half().to(dev)
    ws = ops.gemm_workspace(16, [(hidden, 2 * inter_p), (inter_p, hidden), (hidden, (heads + 2 * kvh) * D)], dev)
    xp = torch.empty(16, hidden, dtype=torch.float16, device=dev)
    ap = torch.empty(16, heads * D, dtype=torch.float16, device=dev)
    xf = x.float().cpu().numpy()
    _close(ops.wo_gemm(x, L["qkv"], ws, x_perm=xp), xf @ np.concatenate([dense["q"], dense["k"], dense["v"]], 1), tol)
    xo = torch.from_numpy(rng.standard_normal((9, heads * D)).astype(np.float32)).half().to(dev)
    _close(ops.wo_gemm(xo, L["o"], ws, x_perm=ap), xo.float().cpu().numpy() @ dense["o"], tol)
    # w13 emits the SiLU*mul output in w2's row order; the padded inter columns stay zero at the end
    act = ops.wo_gemm(x, L["w13"], ws, silu_mul=True, x_perm=xp)
    g, u = xf @ dense["gate"], xf @ dense["up"]
    _close(act[:, :inter], (g / (1 + np.exp(-g)) * u)[:, p2.numpy()], tol)
    assert float(act[:, inter:].abs().max()) == 0.0
    y = ops.wo_gemm(act, L["w2"], ws)
    _close(y, act[:, :inter].float().cpu().numpy() @ dense["down"][p2.numpy()], tol)
    # the fold is the unfolded composition bit for bit: w13 in the checkpoint's column order, gather by w2's order, sorted w2
    w13_plain = ld._groupwise([names["gate"], names["up"]], pad_out=align, gate_up_inter=inter_p)
    act_plain = ops.wo_gemm(x, w13_plain, ws, silu_mul=True, x_perm=xp)
    p2e = torch.cat([p2, torch.arange(inter, inter_p)]).to(torch.int32).to(dev)
    act_gathered = ops.permute_cols(act_plain, p2e)
    assert same_bits(act, act_gathered)
    assert same_bits(y, ops.wo_gemm(act_gathered, L["w2"], ws))


# ---------------------------------------------------------------------------------------------- the whole step
@pytest.mark.parametrize("mode", ["eager", "graph", "graph+pdl", "program", "program+graph+pdl"])
@pytest.mark.parametrize("quant", ["int4", "int8g"])
def test_decode_step_with_act_order_matches_the_oracle(quant, mode):
    check_step(quant=quant, batch=5, ctx=70, mode=mode, act_order=True, seed=2, dev=dev)


# act-order with the other step modes: a verification step (q_len 2) and the Llama-3.1 rope
COMBOS = [(TINY, 2, "eager"), (TINY, 2, "graph+pdl"), (TINY31, 1, "eager")]


@pytest.mark.parametrize("case", COMBOS, ids=["int4 q_len 2 eager", "int4 q_len 2 graph+pdl", "llama31 eager"])
def test_act_order_step_with_verification_or_llama31_rope_matches_the_oracle(case):
    cfg, q_len, mode = case
    check_step(cfg, quant="int4", batch=5, ctx=70, mode=mode, q_len=q_len, act_order=True, seed=2, dev=dev)


def test_act_order_adds_three_gathers_per_layer_and_nothing_when_off():
    cfg = dataclasses.replace(TINY, quant="int4")
    default = DecodeStep(cfg, 3, 40, dev, seed=1)
    off = DecodeStep(cfg, 3, 40, dev, seed=1, act_order=False)
    on = DecodeStep(cfg, 3, 40, dev, seed=1, act_order=True)
    n_default, n_off, n_on = default.launches_per_step(), off.launches_per_step(), on.launches_per_step()
    torch.cuda.synchronize()
    assert n_off == n_default and n_on == n_off + 3 * cfg.layers
    assert same_bits(off.logits, default.logits)
    assert all(L["qkv"].perm is None and L["w13"].perm is None and "perm" not in L for L in off.layers)
