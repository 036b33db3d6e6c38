"""CPU tests: the oracle (oracle/decode_oracle.c via oracle/oracle.py) against the golden vectors produced by the
reference's own Python code (oracle/make_golden.py).  This is what pins the oracle (task section 3)."""
import os

import numpy as np
import pytest

from oracle import oracle as orc


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


@pytest.mark.parametrize("fmt", ["gptq", "awq"])
def test_unpack_groupwise_matches_reference_loader(golden_dir, fmt):
    g = _load(golden_dir, f"quant_unpack_{fmt}.npz")
    qp, zs, sc = orc.unpack_groupwise_int4(g["qweight"], g["qzeros"], g["scales"], int(g["group"]), fmt == "gptq")
    assert np.array_equal(qp, g["q_packed"])                      # bit-exact nibbles
    assert np.array_equal(zs.view(np.uint16), g["zeros_x_scales"].view(np.uint16))  # bit-exact fp16
    assert np.array_equal(sc.view(np.uint16), g["scales_out"].view(np.uint16))


@pytest.mark.parametrize("fmt", ["gptq", "awq"])
def test_unpack_groupwise_8bit_matches_reference_loader(golden_dir, fmt):
    """weight_bits == 8 branch of preprocess_groupwise_weight_params (device_impl.py:256-258), goldens by the reference's code."""
    g = _load(golden_dir, f"quant_unpack8_{fmt}.npz")
    q, zs, sc = orc.unpack_groupwise_int8(g["qweight"], g["qzeros"], g["scales"], int(g["group"]), fmt == "gptq")
    assert q.dtype == np.int8 and np.array_equal(q, g["q"])
    assert np.array_equal(zs.view(np.uint16), g["zeros_x_scales"].view(np.uint16))
    assert np.array_equal(sc.view(np.uint16), g["scales_out"].view(np.uint16))


def test_int8_groupwise_gemm_oracle_consistency():
    """fmt int8g of the C oracle against the numpy dequant formula W' = q_s * s + zeros_x_scales (one rounding) + fp64 matmul."""
    rng = np.random.default_rng(5)
    B, K, N = 3, 256, 96
    x = (rng.standard_normal((B, K)) * 0.5).astype(np.float16)
    q = rng.integers(-128, 128, (K, N), dtype=np.int8)
    s = (np.abs(rng.standard_normal((K // 128, N))) * 6e-4 + 6e-5).astype(np.float16)
    zs = ((128 - rng.integers(0, 256, (K // 128, N))).astype(np.float32) * s.astype(np.float32)).astype(np.float16)
    for fast in (False, True):
        y = orc.from_bits(orc.dequant_gemm(x.view(np.uint16), "int8g", q, scales=s, zeros_x_scales=zs, group=128, fast=fast), False)
        w = orc.dequant_np("int8g", q, s, zs, 128) if not fast else (q.astype(np.float32) * np.repeat(s.astype(np.float32), 128, 0)
                                                                        + np.repeat(zs.astype(np.float32), 128, 0))
        exp = x.astype(np.float64) @ w.astype(np.float64)
        assert np.allclose(y, exp, rtol=2e-3, atol=2e-3), fast


def test_int8_per_column_quantiser_matches_reference(golden_dir):
    g = _load(golden_dir, "quant_int8.npz")
    q, s = orc.quantize_int8_per_col(g["weight"])
    assert np.array_equal(q, g["q"])
    assert np.array_equal(s, g["scale"].astype(np.float32))


@pytest.mark.parametrize("name", ["attn_p16_gqa4", "attn_p64_gqa8", "attn_p32_mha"])
def test_paged_decode_attention_matches_reference_oracle(golden_dir, name):
    g = _load(golden_dir, f"{name}.npz")
    page_list = orc.convert_block_table(g["block_ids"])
    out = orc.paged_decode_attn(g["q"].view(np.uint16), g["kv_pool"].view(np.uint16), page_list,
                                g["sequence_lengths"], int(g["head_num"]), int(g["kv_head_num"]),
                                int(g["head_dim"]), int(g["tokens_per_block"]))
    got = orc.from_bits(out, False)
    # reference tolerance: rtol = atol = 1e-2 (base_attention_test.py:147-148)
    np.testing.assert_allclose(got, g["expect"], rtol=1e-2, atol=1e-2)
    # and the float64 numpy restatement agrees much tighter than that
    ref64 = orc.paged_decode_attn_np(g["q"].astype(np.float64), g["kv_pool"].astype(np.float64), g["block_ids"],
                                     g["sequence_lengths"], int(g["tokens_per_block"]))
    np.testing.assert_allclose(got, ref64, rtol=2e-3, atol=2e-3)


def test_indexing_matches_reference_expected_values(golden_dir):
    g = _load(golden_dir, "indexing.npz")
    got = orc.convert_block_table(g["block_id"])
    assert np.array_equal(got[:, 0], g["kv_offset"])
    assert np.array_equal(orc.convert_block_table_np(g["block_id"]), got)
    for tag in "abcd":
        lens, T = g[f"plan_{tag}_lens"], int(g[f"plan_{tag}_T"])
        nb = [-(-int(L) // T) for L in lens]
        M = max(nb)
        block_ids = np.zeros((len(lens), M), np.int32)
        off = 0
        for b, n in enumerate(nb):
            block_ids[b, :n] = np.arange(off, off + n)
            off += n
        plan = orc.paged_attn_plan(lens - 1, block_ids, T)     # engine passes len-1 (SURVEY a3)
        assert np.array_equal(plan["page_indptr"], g[f"plan_{tag}_indptr"])
        assert np.array_equal(plan["page_indice"], g[f"plan_{tag}_indices"])
        assert np.array_equal(plan["last_page_len"], g[f"plan_{tag}_last"])
        assert np.array_equal(plan["positions"], lens - 1)
        assert np.array_equal(plan["batch_indice"], np.arange(len(lens)))


@pytest.mark.parametrize("fmt", ["f16", "int8", "int4"])
def test_dequant_gemm_c_vs_numpy(fmt):
    rng = np.random.default_rng(7)
    B, K, N, group = 5, 256, 96, 128
    x = (rng.standard_normal((B, K))).astype(np.float16)
    if fmt == "f16":
        w = (rng.standard_normal((K, N)) * 0.05).astype(np.float16)
        wd = orc.dequant_np("f16", w.astype(np.float32))
        y = orc.dequant_gemm(x.view(np.uint16), "f16", w.view(np.uint16))
    elif fmt == "int8":
        q = rng.integers(-128, 128, (K, N)).astype(np.int8)
        s = (np.abs(rng.standard_normal(N)) * 0.01 + 1e-3).astype(np.float16)
        wd = orc.dequant_np("int8", q, s)
        y = orc.dequant_gemm(x.view(np.uint16), "int8", q, scales=s)
    else:
        qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
        s = (np.abs(rng.standard_normal((K // group, N))) * 0.01 + 1e-3).astype(np.float16)
        z = rng.integers(0, 16, (K // group, N))
        zs = ((8 - z).astype(np.float16) * s).astype(np.float16)
        wd = orc.dequant_np("int4", qp, s, zs, group)
        y = orc.dequant_gemm(x.view(np.uint16), "int4", qp, scales=s, zeros_x_scales=zs, group=group)
        yf = orc.dequant_gemm(x.view(np.uint16), "int4", qp, scales=s, zeros_x_scales=zs, group=group, fast=True)
        np.testing.assert_allclose(orc.from_bits(yf, False), orc.from_bits(y, False), rtol=2e-3, atol=2e-3)
    ref = (x.astype(np.float64) @ wd.astype(np.float64)).astype(np.float16).astype(np.float32)
    np.testing.assert_allclose(orc.from_bits(y, False), ref, rtol=1e-3, atol=1e-3)


def test_glue_ops_against_numpy():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((3, 64)).astype(np.float16)
    r = rng.standard_normal((3, 64)).astype(np.float16)
    gmm = rng.standard_normal(64).astype(np.float16)
    y, res = orc.add_rmsnorm(x.view(np.uint16), r.view(np.uint16), gmm.view(np.uint16), 1e-6)
    rr = (x.astype(np.float32) + r.astype(np.float32)).astype(np.float16)
    assert np.array_equal(res.view(np.float16), rr)
    rf = rr.astype(np.float32)
    exp = rf / np.sqrt((rf * rf).mean(-1, keepdims=True) + 1e-6) * gmm.astype(np.float32)
    np.testing.assert_allclose(orc.from_bits(y, False), exp, rtol=2e-3, atol=2e-3)
    gu = rng.standard_normal((3, 32)).astype(np.float16)
    s = orc.silu_and_mul(gu.view(np.uint16))
    gf, uf = gu[:, :16].astype(np.float32), gu[:, 16:].astype(np.float32)
    np.testing.assert_allclose(orc.from_bits(s, False), gf / (1 + np.exp(-gf)) * uf, rtol=2e-3, atol=2e-3)
    lg = rng.standard_normal((4, 1000)).astype(np.float32)
    lg[2, 10] = lg[2, 500] = 99.0
    assert np.array_equal(orc.argmax(lg), lg.argmax(-1).astype(np.int32))


def test_rope_append_roundtrip_properties():
    rng = np.random.default_rng(5)
    B, Hq, Hkv, D, T, M = 2, 4, 2, 128, 16, 3
    qkv = rng.standard_normal((B, (Hq + 2 * Hkv) * D)).astype(np.float16)
    pool = np.zeros((1 + B * M, 2, Hkv, T, D), np.float16)
    block_ids = (np.arange(B * M, dtype=np.int32) + 1).reshape(B, M)
    pl = orc.convert_block_table(block_ids)
    seq = np.array([0, 37], np.int32)
    q, pool2 = orc.rope_append(qkv.view(np.uint16), pool.view(np.uint16), pl, seq, Hq, Hkv, D, T, 500000.0)
    q = q.view(np.float16).reshape(B, Hq, D)
    pool2 = pool2.view(np.float16).reshape(pool.shape)
    # position 0 -> identity rotation
    np.testing.assert_array_equal(q[0], qkv[0, : Hq * D].reshape(Hq, D))
    # rotation preserves the norm of each (i, i+D/2) pair
    src = qkv[1, : Hq * D].reshape(Hq, D).astype(np.float32)
    n0 = src[:, :64] ** 2 + src[:, 64:] ** 2
    n1 = q[1, :, :64].astype(np.float32) ** 2 + q[1, :, 64:].astype(np.float32) ** 2
    np.testing.assert_allclose(n1, n0, rtol=5e-3, atol=5e-3)
    # V copied verbatim to page block_ids[1][37//16], slot 37%16
    v = qkv[1, (Hq + Hkv) * D:].reshape(Hkv, D)
    np.testing.assert_array_equal(pool2[block_ids[1, 2], 1, :, 37 % 16, :], v)
    # nothing else written
    assert np.count_nonzero(pool2) <= 2 * 2 * Hkv * D


@pytest.mark.parametrize("name", ["rope_base10000", "rope_base500000", "rope_d64"])
def test_rope_matches_reference_torch_rope(golden_dir, name):
    """oracle_rope_append pinned to the reference's own pure-torch RoPE (create_cos_sin_cache + apply_rope_reference,
    test_mha_rotary_emb.py:47-81,121-165; fixtures by oracle/make_golden.py). Tolerance = the reference test's
    rtol = atol = 1e-2 (:506-507); V must be appended unrotated, bit for bit."""
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    qkv = g["qkv"]
    B = qkv.shape[0]
    Hq, Hkv, D = int(g["head_num"]), int(g["kv_head_num"]), int(g["head_dim"])
    pos = g["positions"].astype(np.int32)
    T = 16
    M = int(pos.max()) // T + 1
    block_ids = (np.arange(B * M, dtype=np.int32) + 1).reshape(B, M)
    pl = orc.convert_block_table(block_ids)
    pool = np.zeros((1 + B * M, 2, Hkv, T, D), np.float16)
    q_out, pool_out = orc.rope_append(qkv.view(np.uint16), pool.view(np.uint16), pl, pos, Hq, Hkv, D, T, float(g["rope_base"]))
    np.testing.assert_allclose(orc.from_bits(q_out, False).reshape(B, Hq, D), g["q_rope"].astype(np.float32), rtol=1e-2, atol=1e-2)
    pool_f = pool_out.view(np.float16).reshape(pool.shape)
    for b in range(B):
        page, slot = block_ids[b, pos[b] // T], pos[b] % T
        np.testing.assert_allclose(pool_f[page, 0, :, slot].astype(np.float32), g["k_rope"][b].astype(np.float32), rtol=1e-2, atol=1e-2)
        v = qkv[b, (Hq + Hkv) * D:].reshape(Hkv, D)
        assert np.array_equal(pool_f[page, 1, :, slot], v)


def _rope_case(g):
    cfg = {k[4:]: (float(g[k]) if g[k].dtype.kind == "f" else int(g[k])) for k in g.files if k.startswith("cfg_")}
    return cfg, g["qkv"], int(g["head_num"]), int(g["kv_head_num"]), int(g["head_dim"]), g["positions"].astype(np.int32)


@pytest.mark.parametrize("name", ["rope_cache_base_scale2", "rope_cache_yarn"])
def test_rope_ex_cache_and_inline_styles_match_reference(golden_dir, name):
    """oracle_rope_append_ex against the reference's torch RoPE applied with the cos/sin table RopeCache.cc builds (Base with
    linear scale, Yarn). The fixture stores the table rows at the sampled positions (built with the reference's torch calls);
    the oracle's numpy builders must reproduce them, and the op must match (1) through the cache and, for Base, (2) with the
    coefficients computed inline by the formulas of rotary_position_embedding.h. (For Yarn the reference's table and its
    in-kernel formula disagree on which of beta_slow / beta_fast bounds the ramp from below -- RopeCache.cc:57-62 vs
    rotary_position_embedding.h:405-410 --; the decode op uses the table whenever it exists, so the table is what is pinned.)"""
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    cfg, qkv, Hq, Hkv, D, pos = _rope_case(g)
    if cfg["style"] == 1:
        cache = orc.rope_cache_base(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"])
    else:
        cache = orc.rope_cache_yarn(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"], cfg["factor1"], cfg["factor2"],
                                    cfg["extrapolation_factor"], cfg["mscale"])
    assert cache.shape[0] == int(g["cache_positions"])
    np.testing.assert_allclose(cache[pos], g["cache_rows"], atol=2e-3)     # float32 cos/sin of angles up to ~4e3 rad
    B, T = qkv.shape[0], 16
    M = int(pos.max()) // T + 1
    block_ids = (np.arange(B * M, dtype=np.int32) + 1).reshape(B, M)
    pl = orc.convert_block_table(block_ids)
    pool = np.zeros((1 + B * M, 2, Hkv, T, D), np.float16)
    for c in ((cache, None) if cfg["style"] == 1 else (cache,)):
        q_out, pool_out = orc.rope_append_ex(qkv.view(np.uint16), pool.view(np.uint16), pl, pos, Hq, Hkv, D, T, cfg, cos_sin_cache=c)
        np.testing.assert_allclose(orc.from_bits(q_out, False).reshape(B, Hq, D), g["q_rope"].astype(np.float32), rtol=1e-2, atol=1e-2)
        pf = pool_out.view(np.float16).reshape(pool.shape)
        for b in range(B):
            np.testing.assert_allclose(pf[block_ids[b, pos[b] // T], 0, :, pos[b] % T].astype(np.float32),
                                       g["k_rope"][b].astype(np.float32), rtol=1e-2, atol=1e-2)


def test_rope_ex_position_override_bias_logn_and_partial_dim():
    rng = np.random.default_rng(3)
    B, Hq, Hkv, D, T, M = 3, 2, 1, 128, 16, 70
    qkv = rng.standard_normal((B, (Hq + 2 * Hkv) * D)).astype(np.float16)
    bias = (rng.standard_normal((Hq + 2 * Hkv) * D) * 0.1).astype(np.float16)
    seq = np.array([5, 40, 1000], np.int32)
    block_ids = (np.arange(B * M, dtype=np.int32) + 1).reshape(B, M)
    pl = orc.convert_block_table(block_ids)
    pool = np.zeros((1 + B * M, 2, Hkv, T, D), np.float16)
    cfg = dict(style=1, dim=64, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=512, extrapolation_factor=1.0, mscale=1.0)
    pid = np.array([0, 77, 0], np.int32)                  # entry > 0 overrides the position, 0 keeps sequence_lengths
    q, pool_o = orc.rope_append_ex(qkv.view(np.uint16), pool.view(np.uint16), pl, seq, Hq, Hkv, D, T, cfg, bias_bits=bias.view(np.uint16),
                                   position_ids=pid, use_logn=True)
    qf = orc.from_bits(q, False).reshape(B, Hq, D)
    xb = (qkv.astype(np.float32) + bias.astype(np.float32)).astype(np.float16).astype(np.float32).reshape(B, Hq + 2 * Hkv, D)
    for b, p in enumerate((5, 77, 1000)):
        inv = 1.0 / np.power(10000.0, np.arange(0, 64, 2) / 64.0)
        c, s_ = np.cos(p * inv), np.sin(p * inv)
        x = xb[b, 0]
        exp = x.copy()
        exp[:32] = x[:32] * c - x[32:64] * s_
        exp[32:64] = x[32:64] * c + x[:32] * s_
        if p > 512:
            exp *= np.log(p + 1) / np.log(512)            # logn scaling of q beyond max_pos
        np.testing.assert_allclose(qf[b, 0], exp, rtol=2e-3, atol=2e-3)
        # K is appended at slot sequence_lengths[b] (not at the overridden position), V unrotated with the bias added
        pf = pool_o.view(np.float16).reshape(pool.shape)
        page, slot = block_ids[b, seq[b] // T], seq[b] % T
        np.testing.assert_allclose(pf[page, 1, 0, slot].astype(np.float32), xb[b, Hq + Hkv], atol=1e-3)
        assert np.abs(pf[page, 0, 0, slot].astype(np.float32)).sum() > 0


@pytest.mark.parametrize("tag", ["f16_512", "f16_4096", "bf16_512", "bf16_4096"])
def test_norm_ops_match_the_reference_cuda_kernels(golden_dir, tag):
    """oracle_add_rmsnorm against OUTPUTS OF THE KERNELS THE REFERENCE BINDS (flashinfer rmsnorm / fused_add_rmsnorm,
    RegisterBaseBindings.hpp:45-60), captured with flashinfer 0.6.11.post2 on a B200 by tools/make_gpu_golden.py and re-captured bit-identically on an H100: the stored residual must be bit-exact,
    the normalised output may differ by one rounding step of the output type (sum-of-squares order)."""
    g = np.load(os.path.join(golden_dir, "flashinfer_glue_ops.npz"))
    is_bf16 = tag.startswith("bf16")
    x, r, w = (g[f"{tag}_{k}"].view(np.uint16) for k in ("x", "res", "w"))
    y, _ = orc.add_rmsnorm(x, None, w, 1e-6, is_bf16)
    tol = 1.6e-2 if is_bf16 else 2e-3
    np.testing.assert_allclose(orc.from_bits(y, is_bf16), orc.from_bits(g[f"{tag}_rmsnorm"].view(np.uint16), is_bf16), rtol=tol, atol=tol)
    y2, r2 = orc.add_rmsnorm(x, r, w, 1e-6, is_bf16)
    assert np.array_equal(r2, g[f"{tag}_fused_res"].view(np.uint16))
    np.testing.assert_allclose(orc.from_bits(y2, is_bf16), orc.from_bits(g[f"{tag}_fused_y"].view(np.uint16), is_bf16), rtol=tol, atol=tol)
    exact = (y2 == g[f"{tag}_fused_y"].view(np.uint16)).mean()
    assert exact > 0.97, f"only {exact:.3f} of the outputs are bit-identical to flashinfer's"


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_silu_and_mul_matches_the_reference_cuda_kernel(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "flashinfer_glue_ops.npz"))
    is_bf16 = tag == "bf16"
    y = orc.silu_and_mul(g[f"{tag}_gate_up"].view(np.uint16), is_bf16)
    exp = g[f"{tag}_silu_and_mul"].view(np.uint16)
    tol = 1.6e-2 if is_bf16 else 2e-3
    np.testing.assert_allclose(orc.from_bits(y, is_bf16), orc.from_bits(exp, is_bf16), rtol=tol, atol=tol)
    assert (y == exp).mean() > 0.97


def test_qk_rmsnorm_oracle_against_numpy():
    rng = np.random.default_rng(8)
    R, Hq, Hkv, D = 3, 4, 2, 64
    qkv = rng.standard_normal((R, (Hq + 2 * Hkv) * D)).astype(np.float16)
    qg, kg = (1 + 0.1 * rng.standard_normal(D)).astype(np.float16), (1 + 0.1 * rng.standard_normal(D)).astype(np.float16)
    out = orc.from_bits(orc.qk_rmsnorm(qkv.view(np.uint16), qg.view(np.uint16), kg.view(np.uint16), Hq, Hkv, D, 1e-6), False)
    x = qkv.astype(np.float32).reshape(R, Hq + 2 * Hkv, D)
    exp = x.copy()
    for h in range(Hq + Hkv):
        g = (qg if h < Hq else kg).astype(np.float32)
        exp[:, h] = x[:, h] / np.sqrt((x[:, h] ** 2).mean(-1, keepdims=True) + 1e-6) * g
    np.testing.assert_allclose(out.reshape(exp.shape), exp, rtol=2e-3, atol=2e-3)
