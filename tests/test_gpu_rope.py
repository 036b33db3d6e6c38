"""b200_rope_append_ex (the full decode rope contract) against oracle_rope_append_ex, which is pinned to the reference's torch
RoPE / RopeCache tables (tests/test_oracle_golden.py), through the C ABI on an H100."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import RopeConfig  # noqa: E402

dev = torch.device("cuda")
BASE = dict(style=1, dim=128, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=2048, extrapolation_factor=1.0, mscale=1.0)
CASES = [
    ("base", BASE, {}),
    ("base linear scale 4", dict(BASE, scale=4.0), {}),
    ("llama3", dict(BASE, style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192), {}),
    ("yarn inline", dict(BASE, style=5, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13), {}),
    ("yarn cache", dict(BASE, style=5, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13), dict(cache="yarn")),
    ("base cache", dict(BASE, scale=2.0), dict(cache="base")),
    ("dynamic ntk", dict(BASE, style=3, scale=2.0, max_pos=512), {}),
    ("qwen dynamic ntk", dict(BASE, style=4, max_pos=512), {}),
    ("partial dim + bias + position_ids + logn", dict(BASE, dim=64, max_pos=512), dict(bias=True, pid=True, logn=True)),
    ("no rope", dict(BASE, style=0), dict(bias=True)),
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rope_append_ex_vs_oracle(case, dtype):
    name, cfg, opt = case
    is_bf16 = dtype == torch.bfloat16
    rng = np.random.default_rng(len(name))
    B, Hq, Hkv, D, T = 5, 4, 2, 128, 16
    seq = np.array([0, 17, 400, 1500, 3000], np.int32)
    M = int(seq.max()) // T + 1
    qkv = torch.from_numpy(rng.standard_normal((B, (Hq + 2 * Hkv) * D)).astype(np.float32)).to(dtype)
    bias = torch.from_numpy((rng.standard_normal((Hq + 2 * Hkv) * D) * 0.1).astype(np.float32)).to(dtype) if opt.get("bias") else None
    pid = np.array([0, 99, 0, 2500, 0], np.int32) if opt.get("pid") else None
    cache = None
    if opt.get("cache") == "base":
        cache = orc.rope_cache_base(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"])
    elif opt.get("cache") == "yarn":
        cache = orc.rope_cache_yarn(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"], cfg["factor1"], cfg["factor2"],
                                    cfg["extrapolation_factor"], cfg["mscale"])
    block_ids = (np.arange(B * M, dtype=np.int32) + 1).reshape(B, M)
    pl_np = orc.convert_block_table(block_ids)
    pool = torch.zeros(1 + B * M, 2, Hkv, T, D, dtype=dtype, device=dev)
    bits = lambda t: t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    q_exp, pool_exp = orc.rope_append_ex(bits(qkv), bits(pool), pl_np, seq, Hq, Hkv, D, T, cfg, bias_bits=None if bias is None else bits(bias),
                                         position_ids=pid, cos_sin_cache=cache, use_logn=bool(opt.get("logn")), is_bf16=is_bf16)
    q = ops.rope_append_ex(qkv.to(dev), pool, torch.from_numpy(pl_np).to(dev), torch.from_numpy(seq).to(dev), Hq, RopeConfig(**cfg),
                           bias=None if bias is None else bias.to(dev), position_ids=None if pid is None else torch.from_numpy(pid).to(dev),
                           cos_sin_cache=None if cache is None else torch.from_numpy(cache).to(dev), use_logn_attn=bool(opt.get("logn")))
    torch.cuda.synchronize()
    tol = 4e-2 if is_bf16 else 1e-2
    np.testing.assert_allclose(q.float().cpu().numpy(), orc.from_bits(q_exp, is_bf16), rtol=tol, atol=tol)
    np.testing.assert_allclose(pool.float().cpu().numpy(), orc.from_bits(pool_exp, is_bf16).reshape(pool.shape), rtol=tol, atol=tol)


def test_rope_append_ex_base_equals_rope_append():
    """Base style without extras must reproduce b200_rope_append (same positions, same pairing) within a rounding step."""
    g = torch.Generator(device=dev).manual_seed(1)
    B, Hq, Hkv, D, T, M = 4, 8, 2, 128, 64, 3
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, generator=g, device=dev).half()
    seq = torch.tensor([0, 63, 64, 150], dtype=torch.int32, device=dev)
    pl = ops.convert_block_table((torch.arange(B * M, dtype=torch.int32, device=dev) + 1).reshape(B, M))
    p1 = torch.zeros(1 + B * M, 2, Hkv, T, D, dtype=torch.float16, device=dev)
    p2 = torch.zeros_like(p1)
    q1 = ops.rope_append(qkv, p1, pl, seq, Hq, 500000.0)
    q2 = ops.rope_append_ex(qkv, p2, pl, seq, Hq, RopeConfig(**dict(BASE, base=500000.0)))
    torch.cuda.synchronize()
    assert (q1.float() - q2.float()).abs().max().item() <= 4e-3 and (p1.float() - p2.float()).abs().max().item() <= 4e-3


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("with_bias", [False, True])
def test_qk_rmsnorm_vs_oracle(dtype, with_bias):
    """b200_qk_rmsnorm (Qwen3 QK-norm, fused_qk_rmsnorm.cu) against its restatement; v heads must stay untouched."""
    is_bf16 = dtype == torch.bfloat16
    rng = np.random.default_rng(4)
    R, Hq, Hkv, D = 7, 8, 2, 128
    mk = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dtype)
    qkv, qg, kg = mk(R, (Hq + 2 * Hkv) * D), 1 + 0.1 * mk(D), 1 + 0.1 * mk(D)
    qb, kb = (0.1 * mk(D), 0.1 * mk(D)) if with_bias else (None, None)
    bits = lambda t: None if t is None else t.contiguous().view(torch.int16).numpy().view(np.uint16)
    exp = orc.qk_rmsnorm(bits(qkv), bits(qg), bits(kg), Hq, Hkv, D, 1e-6, bits(qb), bits(kb), is_bf16)
    x = qkv.clone().to(dev)
    ops.qk_rmsnorm(x, qg.to(dev), kg.to(dev), Hq, Hkv, D, 1e-6, None if qb is None else qb.to(dev), None if kb is None else kb.to(dev))
    torch.cuda.synchronize()
    tol = 1.6e-2 if is_bf16 else 2e-3
    np.testing.assert_allclose(x.float().cpu().numpy(), orc.from_bits(exp, is_bf16), rtol=tol, atol=tol)
    assert torch.equal(x[:, (Hq + Hkv) * D:].cpu(), qkv[:, (Hq + Hkv) * D:])
