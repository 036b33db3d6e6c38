"""The pybind plugin form of the boundary (rtp_llm_b200/csrc/pybind_ops.cc): `registerPyModuleOps` fills an `rtp_llm_ops`
submodule with an XQAAttnOp-shaped class. CPU part: it builds, imports and exposes the reference's method set; GPU part:
the op runs through the same C ABI and matches the oracle."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

from rtp_llm_b200 import build


def _load():
    path = build.build_pybind()
    spec = importlib.util.spec_from_file_location("b200_compute_ops", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.rtp_llm_ops


def test_pybind_module_exposes_the_reference_surface():
    ops = _load()
    for m in ("support", "prepare", "update", "update_kv_cache_offset", "forward"):      # XQAAttnOp.cc:158-176
        assert hasattr(ops.B200AttnOp, m)
    assert hasattr(ops.B200AttnParams, "kv_cache_offset") and hasattr(ops.B200AttnParams, "__cpp_ptr__")
    cfg = ops.AttentionConfigs()
    cfg.head_num, cfg.kv_head_num, cfg.size_per_head, cfg.tokens_per_block = 32, 8, 128, 64
    inp = ops.PyAttentionInputs()
    inp.is_prefill = True
    assert ops.B200AttnOp(cfg).support(inp) is False       # decode only (and no sm_90 device without a GPU)
    assert issubclass(ops.B200AttnParams, ops.ParamsBase)


def test_pybind_glue_ops_carry_the_reference_names_and_arguments():
    """registerBasicCudaOps (cuda/RegisterBaseBindings.hpp:45-160): same function names and keyword arguments, so a model file
    written against rtp_llm_ops runs unchanged; bad inputs raise (RuntimeError) before anything is launched."""
    ops = _load()
    want = {"rmsnorm": ("output", "input", "weight", "eps", "cuda_stream"),
            "fused_add_rmsnorm": ("input", "residual", "weight", "eps", "cuda_stream"),
            "silu_and_mul": ("output", "input", "cuda_stream"),
            "fused_qk_rmsnorm": ("IO", "q_gamma", "k_gamma", "layernorm_eps", "q_group_num", "k_group_num", "m", "n", "norm_size"),
            "embedding": ("output", "input", "weight", "position_ids", "token_type_ids", "text_tokens_mask")}
    for name, args in want.items():
        doc = getattr(ops, name).__doc__
        sig = doc[doc.index("(") + 1:doc.index(") ->")]
        names = tuple(part.split(":")[0].strip() for part in sig.split(", ") if ":" in part)
        assert names == args, (name, doc)
    x = torch.zeros(2, 64, dtype=torch.float16)            # CPU tensors: rejected by the wrapper's checks
    with pytest.raises(RuntimeError):
        ops.rmsnorm(x.clone(), x, torch.ones(64, dtype=torch.float16), 1e-6)
    with pytest.raises(RuntimeError):
        ops.silu_and_mul(x.clone(), x)


@pytest.mark.gpu
def test_pybind_glue_ops_match_oracle():
    from oracle import oracle as orc
    ops = _load()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    bits = lambda t: t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    for dtype in (torch.float16, torch.bfloat16):
        is_bf16 = dtype == torch.bfloat16
        tol = 2e-2 if is_bf16 else 4e-3
        rows, hidden = 5, 1024
        x = torch.randn(rows, hidden, generator=g, device=dev).to(dtype)
        r = torch.randn(rows, hidden, generator=g, device=dev).to(dtype)
        w = (1 + 0.1 * torch.randn(hidden, generator=g, device=dev)).to(dtype)
        sid = torch.cuda.current_stream().cuda_stream
        # rmsnorm(output, input, weight, eps, cuda_stream)
        y = torch.empty_like(x)
        ops.rmsnorm(y, x, w, 1e-6, sid)
        y_e, _ = orc.add_rmsnorm(bits(x), None, bits(w), 1e-6, is_bf16)
        np.testing.assert_allclose(y.float().cpu().numpy(), orc.from_bits(y_e, is_bf16), rtol=tol, atol=tol)
        # fused_add_rmsnorm(input, residual, weight, eps, cuda_stream): both updated in place
        x2, r2 = x.clone(), r.clone()
        ops.fused_add_rmsnorm(x2, r2, w, 1e-6, sid)
        y_e, r_e = orc.add_rmsnorm(bits(x), bits(r), bits(w), 1e-6, is_bf16)
        torch.cuda.synchronize()
        assert np.array_equal(bits(r2), r_e)                                  # the stored residual is bit-exact
        np.testing.assert_allclose(x2.float().cpu().numpy(), orc.from_bits(y_e, is_bf16), rtol=tol, atol=tol)
        # silu_and_mul(output, input, cuda_stream)
        gu = torch.randn(rows, 2 * 384, generator=g, device=dev).to(dtype)
        act = torch.empty(rows, 384, device=dev, dtype=dtype)
        ops.silu_and_mul(act, gu)
        np.testing.assert_allclose(act.float().cpu().numpy(), orc.from_bits(orc.silu_and_mul(bits(gu), is_bf16), is_bf16), rtol=tol, atol=tol)
        # fused_qk_rmsnorm(IO, q_gamma, k_gamma, eps, q_group_num, k_group_num, m, n, norm_size): in place, v heads untouched
        Hq, Hkv, D = 4, 2, 128
        qkv = torch.randn(rows, (Hq + 2 * Hkv) * D, generator=g, device=dev).to(dtype)
        qg = (1 + 0.1 * torch.randn(D, generator=g, device=dev)).to(dtype)
        kg = (1 + 0.1 * torch.randn(D, generator=g, device=dev)).to(dtype)
        exp = orc.qk_rmsnorm(bits(qkv), bits(qg), bits(kg), Hq, Hkv, D, 1e-6, is_bf16=is_bf16)
        ops.fused_qk_rmsnorm(qkv, qg, kg, 1e-6, Hq, Hkv, rows, qkv.shape[1], D)
        np.testing.assert_allclose(qkv.float().cpu().numpy(), orc.from_bits(exp, is_bf16), rtol=tol, atol=tol)
        # embedding(output, input, weight)
        table = torch.randn(50, 256, generator=g, device=dev).to(dtype)
        ids = torch.tensor([3, 49, 0, 3], dtype=torch.int32, device=dev)
        out = torch.empty(4, 256, device=dev, dtype=dtype)
        ops.embedding(out, ids, table)
        assert torch.equal(out, table[ids.long()])
    with pytest.raises(RuntimeError):
        ops.fused_qk_rmsnorm(qkv, qg, kg, 1e-6, Hq, Hkv, rows, qkv.shape[1], 64)   # n != (q + 2k) * norm_size


@pytest.mark.gpu
def test_pybind_attn_and_linear_ops_match_oracle():
    from oracle import oracle as orc
    from rtp_llm_b200 import ops as b200ops
    from rtp_llm_b200._lib import B200_FMT_INT4
    ops = _load()
    dev = torch.device("cuda")
    torch.manual_seed(42)
    B, Hq, Hkv, D, T = 4, 8, 2, 128, 64
    lens = [63, 64, 200, 511]
    M = max(math.ceil((L + 1) / T) for L in lens)
    P = B * M + 1
    pool = torch.randn(P, 2, Hkv, T, D, device=dev).half()
    block_ids = (torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M)
    seq = torch.tensor(lens, dtype=torch.int32, device=dev)
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, device=dev).half()
    cfg = ops.AttentionConfigs()
    cfg.head_num, cfg.kv_head_num, cfg.size_per_head, cfg.tokens_per_block = Hq, Hkv, D, T
    cfg.max_seq_len = M * T
    cfg.rope_config.base = 500000.0
    inp = ops.PyAttentionInputs()
    inp.sequence_lengths, inp.kv_cache_kernel_block_id_device = seq, block_ids
    op = ops.B200AttnOp(cfg)
    assert op.support(inp)
    params = op.prepare(inp)
    kv = ops.LayerKVCache()
    kv.kv_cache_base = pool
    pool0 = pool.clone()
    q = ops.b200_rope_kvcache_decode(qkv, kv, params, cfg)
    out = op.forward(q, kv, params)
    torch.cuda.synchronize()
    bits = lambda t: t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    pl = orc.convert_block_table(block_ids.cpu().numpy())
    assert np.array_equal(params.kv_cache_offset.cpu().numpy(), pl)
    q_e, pool_e = orc.rope_append(bits(qkv), bits(pool0), pl, np.array(lens, np.int32), Hq, Hkv, D, T, 500000.0)
    out_e = orc.paged_decode_attn(q_e.reshape(B, Hq, D), pool_e, pl, np.array(lens, np.int32), Hq, Hkv, D, T)
    np.testing.assert_allclose(out.float().cpu().numpy(), orc.from_bits(out_e, False), rtol=1e-2, atol=1e-2)
    # update(): new block table, refreshed in place
    inp2 = ops.PyAttentionInputs()
    inp2.sequence_lengths, inp2.kv_cache_kernel_block_id_device = seq, block_ids.flip(0).contiguous()
    op.update(params, inp2)
    torch.cuda.synchronize()
    assert np.array_equal(params.kv_cache_offset.cpu().numpy(), orc.convert_block_table(inp2.kv_cache_kernel_block_id_device.cpu().numpy()))
    with pytest.raises(RuntimeError):
        op.forward(q, None, params)                         # "decode should have kv cache."
    # linear op on a packed INT4 weight
    rng = np.random.default_rng(1)
    K, N = 256, 256
    qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
    s = (np.abs(rng.standard_normal((K // 128, N))) * 0.01 + 1e-3).astype(np.float16)
    zs = ((8 - rng.integers(0, 16, (K // 128, N))).astype(np.float16) * s).astype(np.float16)
    pw = b200ops.pack_w4(torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dev), torch.from_numpy(zs).to(dev))
    lin = ops.B200LinearOp(B200_FMT_INT4, K, N, pw.data)
    x = torch.randn(5, K, device=dev).half()
    y = lin.forward(x)
    exp = orc.dequant_gemm(bits(x), "int4", qp, scales=s, zeros_x_scales=zs, group=128)
    np.testing.assert_allclose(y.float().cpu().numpy(), orc.from_bits(exp, False), rtol=2e-2, atol=2e-2)
