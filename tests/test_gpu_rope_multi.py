"""GPU tests (H100) of the full rope contract for several tokens per sequence and through the attention seams:
b200_rope_append_ex_multi against successive one-token calls, B200DecodeImpl and the pybind B200AttnOp against the op-by-op
oracle for each rope style at q_len 1 and 3, and a DecodeStep under a Llama-3.1 rope config (verification steps and decode
programs included) against the step oracle."""
import ctypes
import importlib.util
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import _lib, attention, build, ops  # noqa: E402
from rtp_llm_b200._lib import RopeConfig  # noqa: E402
from tests.step_oracle import TINY31, check_step  # noqa: E402
from tests.test_gpu_rope import CASES  # noqa: E402

DEV = torch.device("cuda")


def _u16(t):
    return t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _oracle_table(cfg, opt):
    if opt.get("cache") == "base":
        return orc.rope_cache_base(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"])
    if opt.get("cache") == "yarn":
        return orc.rope_cache_yarn(cfg["dim"], cfg["base"], cfg["scale"], cfg["max_pos"], cfg["factor1"], cfg["factor2"],
                                   cfg["extrapolation_factor"], cfg["mscale"])
    return None


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("q_len", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rope_append_ex_multi_equals_single_token_calls(case, dtype, q_len):
    """Token j of a q_len call has the bits of a one-token call at sequence_lengths + j: q rows and the whole KV pool. Page
    size 16 with sequences cached up to 15 and 1502 tokens: every step crosses a page boundary."""
    name, cfg, opt = case
    g = torch.Generator(device=DEV).manual_seed(len(name) + q_len)
    B, Hq, Hkv, D, T = 4, 4, 2, 128, 16
    lens = [0, 15, 1502, 3000]
    M = max(-(-(L + q_len) // T) for L in lens)
    P = B * M + 1
    pool1 = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    pool2 = pool1.clone()
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    bias = (0.1 * torch.randn((Hq + 2 * Hkv) * D, generator=g, device=DEV)).to(dtype) if opt.get("bias") else None
    pid = None
    if opt.get("pid"):     # zero (keep the slot), inside max_pos, and past max_pos (logn) entries, per row
        pid = torch.tensor([[0, 99 + j, 2500 + j, 0][b] for b in range(B) for j in range(q_len)], dtype=torch.int32, device=DEV)
        pid[1::3] = 0
    cache = _oracle_table(cfg, opt)
    cache = None if cache is None else torch.from_numpy(cache).to(DEV)
    pl = ops.convert_block_table((torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1).reshape(B, M))
    seq = torch.tensor(lens, dtype=torch.int32, device=DEV)
    kw = dict(bias=bias, cos_sin_cache=cache, use_logn_attn=bool(opt.get("logn")))
    rc = RopeConfig(**cfg)
    q = ops.rope_append_ex(qkv, pool1, pl, seq, Hq, rc, position_ids=pid, q_len=q_len, **kw).view(B, q_len, -1)
    rows = qkv.view(B, q_len, -1)
    for j in range(q_len):
        pj = None if pid is None else pid.view(B, q_len)[:, j].contiguous()
        qj = ops.rope_append_ex(rows[:, j].contiguous(), pool2, pl, seq + j, Hq, rc, position_ids=pj, **kw)
        assert torch.equal(q[:, j], qj), f"q of token {j} differs"
    torch.cuda.synchronize()
    assert torch.equal(pool1, pool2), "cache contents differ"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rope_append_ex_multi_at_one_token_is_rope_append_ex(case, dtype):
    name, cfg, opt = case
    g = torch.Generator(device=DEV).manual_seed(len(name))
    B, Hq, Hkv, D, T, M = 5, 4, 2, 128, 16, 200
    P = B * M + 1
    pool1 = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    pool2 = pool1.clone()
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    bias = (0.1 * torch.randn((Hq + 2 * Hkv) * D, generator=g, device=DEV)).to(dtype) if opt.get("bias") else None
    pid = torch.tensor([0, 99, 0, 2500, 0], dtype=torch.int32, device=DEV) if opt.get("pid") else None
    cache = _oracle_table(cfg, opt)
    cache = None if cache is None else torch.from_numpy(cache).to(DEV)
    pl = ops.convert_block_table((torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1).reshape(B, M))
    seq = torch.tensor([0, 17, 400, 1500, 3000], dtype=torch.int32, device=DEV)
    rc = RopeConfig(**cfg)
    logn = bool(opt.get("logn"))
    q1 = ops.rope_append_ex(qkv, pool1, pl, seq, Hq, rc, bias=bias, position_ids=pid, cos_sin_cache=cache, use_logn_attn=logn)
    q2 = torch.empty_like(q1)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    rc_p = ctypes.cast(ctypes.pointer(rc), ctypes.c_void_p)
    rcode = _lib.load().b200_rope_append_ex_multi(p(qkv), p(bias), p(q2), p(pool2), p(pl), p(seq), p(pid), p(cache),
                                                  0 if cache is None else cache.shape[0], rc_p, int(logn),
                                                  int(dtype == torch.bfloat16), B, Hq, Hkv, D, M, T, 1,
                                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rcode == 0, _lib.load().b200_last_error()
    torch.cuda.synchronize()
    assert torch.equal(q1, q2) and torch.equal(pool1, pool2)


# ------------------------------------------------------------------------------------------------------------ seams
def _pybind():
    spec = importlib.util.spec_from_file_location("b200_compute_ops", build.build_pybind())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.rtp_llm_ops


BASE = dict(style=1, dim=128, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=2048, extrapolation_factor=1.0, mscale=1.0)
# name, rope config, use_logn_attn, position ids, oracle table
SEAM = [
    ("llama3", dict(BASE, style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192), False, False, None),
    ("yarn table", dict(BASE, style=5, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13), False, False, "yarn"),
    ("base linear scale table", dict(BASE, scale=2.0, max_pos=1024), False, False, "base"),
    ("dynamic ntk", dict(BASE, style=3, scale=2.0, max_pos=512), False, False, None),
    ("partial dim + logn + position ids", dict(BASE, dim=64, max_pos=512), True, True, "base"),
]


def _seam_case(B, q_len, Hq, Hkv, D, T, lens, dtype, seed, with_pid):
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = max(-(-(L + q_len) // T) for L in lens)
    P = B * M + 1
    pool = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    block_ids = (torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1).reshape(B, M)
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    seq = torch.tensor(lens, dtype=torch.int32, device=DEV)
    pid = None
    if with_pid:
        pid = torch.tensor([(0 if b % 2 == 0 else 600 + 7 * b) + (j if b % 2 else 0) for b in range(B) for j in range(q_len)],
                           dtype=torch.int32, device=DEV)
    return pool, block_ids, qkv, seq, pid, M


def _run_python_seam(fields, logn, pool, block_ids, qkv, seq, pid, q_len, Hq, Hkv, D, T, M):
    cfg = SimpleNamespace(head_num=Hq, kv_head_num=Hkv, size_per_head=D, tokens_per_block=T, max_seq_len=M * T, q_scaling=1.0,
                          need_rope_kv_cache=True, use_logn_attn=logn,
                          rope_config=None if fields is None else SimpleNamespace(**fields))
    inp = SimpleNamespace(is_prefill=False, sequence_lengths=seq, kv_cache_kernel_block_id_device=block_ids,
                          input_lengths=torch.full((seq.shape[0],), q_len, dtype=torch.int32), combo_position_ids=pid)
    assert attention.B200DecodeImpl.support(cfg, inp)
    impl = attention.B200DecodeImpl(cfg, inp)
    return impl.forward(qkv, pool)


def _run_pybind_seam(m, fields, logn, pool, block_ids, qkv, seq, pid, q_len, Hq, Hkv, D, T, M):
    cfg = m.AttentionConfigs()
    cfg.head_num, cfg.kv_head_num, cfg.size_per_head, cfg.tokens_per_block, cfg.max_seq_len = Hq, Hkv, D, T, M * T
    cfg.use_logn_attn = logn
    if fields is not None:
        r = m.RopeConfig()
        for k, v in fields.items():
            setattr(r, k, v)
        cfg.rope_config = r
    inp = m.PyAttentionInputs()
    inp.sequence_lengths, inp.kv_cache_kernel_block_id_device = seq, block_ids
    inp.input_lengths = torch.full((seq.shape[0],), q_len, dtype=torch.int32)
    if pid is not None:
        inp.combo_position_ids = pid
    op = m.B200AttnOp(cfg)
    assert op.support(inp)
    params = op.prepare(inp)
    kv = m.LayerKVCache()
    kv.kv_cache_base = pool
    q = m.b200_rope_kvcache_decode(qkv, kv, params, cfg)
    return op.forward(q, kv, params)


@pytest.mark.parametrize("q_len", [1, 3])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", SEAM, ids=[c[0] for c in SEAM])
def test_seams_match_the_oracle_per_rope_style(case, dtype, q_len):
    name, fields, logn, with_pid, table = case
    is_bf16 = dtype == torch.bfloat16
    B, Hq, Hkv, D, T = 4, 8, 2, 128, 16
    lens = [0, 30, 700, 1500]
    pool, block_ids, qkv, seq, pid, M = _seam_case(B, q_len, Hq, Hkv, D, T, lens, dtype, len(name), with_pid)
    pool0 = pool.clone()
    pool_py, pool_pb = pool.clone(), pool.clone()
    out_py = _run_python_seam(fields, logn, pool_py, block_ids, qkv, seq, pid, q_len, Hq, Hkv, D, T, M)
    out_pb = _run_pybind_seam(_pybind(), fields, logn, pool_pb, block_ids, qkv, seq, pid, q_len, Hq, Hkv, D, T, M)
    torch.cuda.synchronize()
    assert torch.equal(out_py, out_pb) and torch.equal(pool_py, pool_pb), "the two seams differ"
    # oracle: the one-token rope contract per token j at seq + j, every K/V appended before any query attends
    cache = _oracle_table(fields, {"cache": table}) if table else None
    pl = orc.convert_block_table(block_ids.cpu().numpy())
    seq_np, qkv_b = seq.cpu().numpy(), _u16(qkv).reshape(B, q_len, -1)
    pid_np = None if pid is None else pid.cpu().numpy().reshape(B, q_len)
    pb, qs = _u16(pool0), []
    for j in range(q_len):
        qj, pb = orc.rope_append_ex(np.ascontiguousarray(qkv_b[:, j]), pb, pl, seq_np + j, Hq, Hkv, D, T, fields,
                                    position_ids=None if pid_np is None else np.ascontiguousarray(pid_np[:, j]), cos_sin_cache=cache,
                                    use_logn=logn, is_bf16=is_bf16)
        qs.append(qj)
    tol = 2e-2 if is_bf16 else 1e-2
    np.testing.assert_allclose(pool_py.float().cpu().numpy(), orc.from_bits(pb, is_bf16).reshape(pool.shape), rtol=tol, atol=tol)
    got = out_py.float().cpu().numpy().reshape(B, q_len, -1)
    for j in range(q_len):
        exp = orc.from_bits(orc.paged_decode_attn(qs[j].reshape(B, Hq, D), pb, pl, seq_np + j, Hq, Hkv, D, T, is_bf16=is_bf16), is_bf16)
        np.testing.assert_allclose(got[:, j], exp, rtol=tol, atol=tol, err_msg=f"query token {j}")


@pytest.mark.parametrize("q_len", [1, 3])
def test_base_only_config_keeps_the_bits_of_rope_append(q_len):
    B, Hq, Hkv, D, T = 3, 8, 2, 128, 32
    pool, block_ids, qkv, seq, _, M = _seam_case(B, q_len, Hq, Hkv, D, T, [5, 31, 400], torch.float16, 3, False)
    fields = dict(base=500000.0)
    pool_ref, pool_py, pool_pb = pool.clone(), pool.clone(), pool.clone()
    out_py = _run_python_seam(fields, False, pool_py, block_ids, qkv, seq, None, q_len, Hq, Hkv, D, T, M)
    out_pb = _run_pybind_seam(_pybind(), fields, False, pool_pb, block_ids, qkv, seq, None, q_len, Hq, Hkv, D, T, M)
    pl = ops.convert_block_table(block_ids)
    q = ops.rope_append(qkv, pool_ref, pl, seq, Hq, 500000.0, q_len=q_len)
    ws = ops.attn_workspace(B * q_len, Hq, Hkv, M * T, DEV)
    if q_len == 1:
        ref = ops.paged_decode_attn(q, pool_ref, pl, seq, min(M * T + 1, M * T), ws)
    else:
        ref = ops.paged_decode_attn_multi(q.view(B, q_len, Hq, D), pool_ref, pl, seq, M * T, ws).reshape(B * q_len, -1)
    torch.cuda.synchronize()
    assert torch.equal(pool_ref, pool_py) and torch.equal(pool_ref, pool_pb)
    assert torch.equal(ref, out_py) and torch.equal(ref, out_pb)


def test_pybind_seam_serves_group_32_and_refuses_unserved_rope():
    m = _pybind()
    B, Hq, Hkv, D, T = 2, 32, 1, 128, 64
    pool, block_ids, qkv, seq, _, M = _seam_case(B, 1, Hq, Hkv, D, T, [70, 300], torch.float16, 5, False)
    pool0 = pool.clone()
    fields = dict(BASE, style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192)
    out = _run_pybind_seam(m, fields, False, pool, block_ids, qkv, seq, None, 1, Hq, Hkv, D, T, M)
    torch.cuda.synchronize()
    pl = orc.convert_block_table(block_ids.cpu().numpy())
    q_e, pool_e = orc.rope_append_ex(_u16(qkv), _u16(pool0), pl, seq.cpu().numpy(), Hq, Hkv, D, T, fields)
    exp = orc.from_bits(orc.paged_decode_attn(q_e.reshape(B, Hq, D), pool_e, pl, seq.cpu().numpy(), Hq, Hkv, D, T), False)
    np.testing.assert_allclose(out.float().cpu().numpy(), exp, rtol=1e-2, atol=1e-2)
    cfg = m.AttentionConfigs()
    cfg.head_num, cfg.kv_head_num, cfg.size_per_head, cfg.tokens_per_block = 32, 8, 128, 64
    inp = m.PyAttentionInputs()
    inp.sequence_lengths, inp.kv_cache_kernel_block_id_device = seq, block_ids
    assert m.B200AttnOp(cfg).support(inp)
    for style, neox, dim in ((2, True, 0), (7, True, 0), (9, True, 0), (1, False, 0), (1, True, 63), (1, True, 256)):
        cfg.rope_config.style, cfg.rope_config.is_neox_style, cfg.rope_config.dim = style, neox, dim
        assert not m.B200AttnOp(cfg).support(inp), (style, neox, dim)
    cfg.need_rope_kv_cache = False                      # the rope config does not matter when the seam does not apply it
    assert m.B200AttnOp(cfg).support(inp)
    inp.input_lengths = torch.full((B,), 16, dtype=torch.int32)  # group 4 x q_len 16 = 64 rows: served
    assert m.B200AttnOp(cfg).support(inp)
    inp.input_lengths = torch.full((B,), 17, dtype=torch.int32)  # 68 rows > 64
    assert not m.B200AttnOp(cfg).support(inp)


# ------------------------------------------------------------------------------------------------------------ step
# program: rope_append_ex is recorded as its own launch between the persistent-kernel segments
STEP = [(1, "eager"), (2, "eager"), (4, "eager"), (4, "graph pdl"), (1, "graph pdl"), (1, "program"), (1, "program graph pdl")]


@pytest.mark.parametrize("case", STEP, ids=[f"q_len {n} {m}" for n, m in STEP])
def test_llama31_step_vs_oracle(case):
    q_len, mode = case
    check_step(TINY31, batch=3, ctx=40, mode=mode, q_len=q_len, dev=DEV)
