"""GPU tests (H100) of QK-RMSNorm fused into RoPE + K/V append (b200_qk_norm_rope_append(_ex)): q_out and the whole K/V pool
bit for bit against the two-launch composition b200_qk_rmsnorm (on a copy of qkv) + b200_rope_append(_ex), for every served
style, head size and grouping, one and several tokens per sequence, eager, under a CUDA graph with PDL behind the qkv GEMM and
recorded in a decode program; v columns copied bit for bit; qkv only read."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import _lib, ops, rope  # noqa: E402
from rtp_llm_b200.rope import RopeSpec  # noqa: E402

DEV = torch.device("cuda")
EPS = 1e-6
T = 16
LENS = [0, 15, 250, 1000]       # ragged; with T 16 every q_len >= 2 crosses a page boundary somewhere


def _spec(style: str, D: int) -> tuple:
    """(RopeSpec, use_logn, with position ids) of a named case at head size D."""
    return {
        "no rope": (RopeSpec(style=rope.NO, dim=D), False, False),
        "plain base": (RopeSpec(dim=D, base=1000000.0), False, False),
        "base table": (RopeSpec(dim=D, base=10000.0, scale=2.0, max_pos=1024), False, False),
        "llama3": (RopeSpec(style=rope.LLAMA3, dim=D, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=512), False, False),
        "yarn table": (RopeSpec(style=rope.YARN, dim=D, base=1000000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=512,
                                mscale=1.14), False, False),
        "dynamic ntk": (RopeSpec(style=rope.DYNAMIC_NTK, dim=D, scale=2.0, max_pos=512), False, False),
        "qwen dynamic ntk": (RopeSpec(style=rope.QWEN_DYNAMIC_NTK, dim=D, max_pos=512), False, False),
        "partial dim + position_ids + logn": (RopeSpec(dim=D // 2, max_pos=512), True, True),
    }[style]


STYLES = ["no rope", "plain base", "base table", "llama3", "yarn table", "dynamic ntk", "qwen dynamic ntk",
          "partial dim + position_ids + logn"]


def _case(B, q_len, Hq, Hkv, D, dtype, seed, with_pid):
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = max(-(-(L + q_len) // T) for L in LENS[:B])
    P = B * M + 1
    pool = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    pl = ops.convert_block_table((torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1).reshape(B, M))
    qkv = (3 * torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV)).to(dtype)
    qg = (1 + 0.3 * torch.randn(D, generator=g, device=DEV)).to(dtype)
    kg = (1 + 0.3 * torch.randn(D, generator=g, device=DEV)).to(dtype)
    seq = torch.tensor(LENS[:B], dtype=torch.int32, device=DEV)
    pid = None
    if with_pid:        # zero (keep the slot), inside max_pos, and past max_pos (logn) entries
        pid = torch.tensor([[0, 99 + j, 700 + j, 0][b] for b in range(B) for j in range(q_len)], dtype=torch.int32, device=DEV)
    return pool, pl, qkv, qg, kg, seq, pid


def _composition(spec, logn, pid, qkv, qg, kg, pool, pl, seq, Hq, Hkv, D, q_len):
    normed = ops.qk_rmsnorm(qkv.clone(), qg, kg, Hq, Hkv, D, EPS)
    return rope.rope_append(spec, normed, pool, pl, seq, Hq, q_len=q_len, use_logn_attn=logn, position_ids=pid)


def _check(style, dtype, D, Hq, Hkv, q_len, B=4):
    spec, logn, with_pid = _spec(style, D)
    pool, pl, qkv, qg, kg, seq, pid = _case(B, q_len, Hq, Hkv, D, dtype, len(style) * 31 + D + Hq + q_len, with_pid)
    qkv0, pool_ref = qkv.clone(), pool.clone()
    q = rope.rope_append(spec, qkv, pool, pl, seq, Hq, q_len=q_len, use_logn_attn=logn, position_ids=pid, qk_norm=(qg, kg, EPS))
    q_ref = _composition(spec, logn, pid, qkv, qg, kg, pool_ref, pl, seq, Hq, Hkv, D, q_len)
    torch.cuda.synchronize()
    assert torch.equal(qkv, qkv0), "qkv was written"
    assert torch.equal(q, q_ref), "q_out differs from qk_rmsnorm + rope_append"
    assert torch.equal(pool, pool_ref), "K/V pool differs from qk_rmsnorm + rope_append"
    return q, pool, qkv, pl, seq


@pytest.mark.parametrize("q_len", [1, 2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("style", STYLES)
def test_fused_equals_norm_then_rope_per_style(style, dtype, q_len):
    _check(style, dtype, 128, 32, 8, q_len)


SHAPES = [(32, 8), (8, 1), (64, 8)]


@pytest.mark.parametrize("q_len", [1, 4])
@pytest.mark.parametrize("style", ["plain base", "yarn table", "partial dim + position_ids + logn"])
@pytest.mark.parametrize("heads", SHAPES, ids=[f"{a}-{b}" for a, b in SHAPES])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_fused_equals_norm_then_rope_per_shape(dtype, D, heads, style, q_len):
    _check(style, dtype, D, heads[0], heads[1], q_len)


@pytest.mark.parametrize("style", ["plain base", "yarn table"])
def test_v_columns_are_copied_bit_for_bit(style):
    B, q_len, Hq, Hkv, D = 4, 4, 8, 2, 128
    _, pool, qkv, pl, seq = _check(style, torch.bfloat16, D, Hq, Hkv, q_len, B)
    v = qkv.view(B, q_len, Hq + 2 * Hkv, D)[:, :, Hq + Hkv:]
    plc, seqc = pl.cpu(), seq.cpu()
    for b in range(B):
        for j in range(q_len):
            slot = int(seqc[b]) + j
            page = int(plc[b, 0, 1, slot // T])
            assert torch.equal(pool.view(-1, Hkv, T, D)[page, :, slot % T], v[b, j]), (b, j)   # page ids count K and V pages


def test_argument_checks():
    lib = _lib.load()
    x = torch.zeros(1024, dtype=torch.float16, device=DEV)
    seq = torch.zeros(1, dtype=torch.int32, device=DEV)
    p = x.data_ptr()
    # null gamma, head sizes that are not a multiple of 64 or exceed 256
    assert lib.b200_qk_norm_rope_append(p, None, p, EPS, p, p, seq.data_ptr(), seq.data_ptr(), 0, 1, 1, 1, 128, 1, 16, 1e6, 1, None) != 0
    assert b"gamma" in lib.b200_last_error()
    for D in (96, 512):
        assert lib.b200_qk_norm_rope_append(p, p, p, EPS, p, p, seq.data_ptr(), seq.data_ptr(), 0, 1, 1, 1, D, 1, 16, 1e6, 1, None) != 0
        assert b"head_dim" in lib.b200_last_error()
    rc = _lib.RopeConfig(style=1, dim=128, base=1e6, scale=1.0, max_pos=0, extrapolation_factor=1.0, mscale=1.0)
    import ctypes
    rcp = ctypes.cast(ctypes.pointer(rc), ctypes.c_void_p)
    assert lib.b200_qk_norm_rope_append_ex(p, p, None, EPS, p, p, seq.data_ptr(), seq.data_ptr(), None, None, 0, rcp, 0, 0, 1, 1, 1,
                                           128, 1, 16, 1, None) != 0
    assert lib.b200_qk_norm_rope_append_ex(p, p, p, EPS, p, p, seq.data_ptr(), seq.data_ptr(), None, None, 0, rcp, 0, 0, 1, 1, 1,
                                           128, 1, 16, 0, None) != 0
    assert b"q_len" in lib.b200_last_error()


def _gemm_case(dtype, q_len, Hq=8, Hkv=2, D=128, K=512, B=4):
    g = torch.Generator(device=DEV).manual_seed(7 + q_len)
    R = B * q_len
    N = (Hq + 2 * Hkv) * D
    qp = torch.randint(0, 256, (K, N // 2), generator=g, device=DEV, dtype=torch.uint8)       # INT4 g128, as the decode step's
    s = (torch.randn(K // 128, N, generator=g, device=DEV).abs() * 0.01 + 1e-3).to(dtype)
    w = ops.pack_w4(qp, s, (-8 * s).to(dtype))
    x = torch.randn(R, K, generator=g, device=DEV).to(dtype)
    ws = ops.gemm_workspace(R, [(K, N)], DEV)
    qkv = torch.empty(R, N, dtype=dtype, device=DEV)
    q = torch.empty(R, Hq * D, dtype=dtype, device=DEV)
    pool, pl, _, qg, kg, seq, _ = _case(B, q_len, Hq, Hkv, D, dtype, 11 + q_len, False)
    return w, x, ws, qkv, q, pool, pl, qg, kg, seq, Hq, Hkv, D


@pytest.mark.parametrize("q_len", [1, 4])
@pytest.mark.parametrize("style", ["plain base", "yarn table"])
def test_same_bits_under_cuda_graph_with_pdl_behind_the_qkv_gemm(style, q_len):
    dtype = torch.bfloat16
    w, x, ws, qkv, q, pool, pl, qg, kg, seq, Hq, Hkv, D = _gemm_case(dtype, q_len)
    spec, _, _ = _spec(style, D)
    rope.table(spec, DEV)
    pool0 = pool.clone()

    def step():
        ops.wo_gemm(x, w, ws, out=qkv, pdl=True)
        rope.rope_append(spec, qkv, pool, pl, seq, Hq, q_out=q, q_len=q_len, qk_norm=(qg, kg, EPS))
    ops.set_pdl(True)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        pool.copy_(pool0)
        q.fill_(0)
        qkv.fill_(0)
        graph.replay()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)
    pool_ref = pool0.clone()
    q_ref = _composition(spec, False, None, qkv, qg, kg, pool_ref, pl, seq, Hq, Hkv, D, q_len)
    torch.cuda.synchronize()
    assert torch.equal(q, q_ref) and torch.equal(pool, pool_ref)


@pytest.mark.parametrize("style", ["plain base", "yarn table"])
def test_same_bits_recorded_in_a_decode_program(style):
    """The fused entry is its own launch inside a program (the persistent kernel's rope op does not normalise), after a qkv
    GEMM that runs inside the persistent kernel."""
    dtype = torch.float16
    w, x, ws, qkv, q, pool, pl, qg, kg, seq, Hq, Hkv, D = _gemm_case(dtype, 1)
    spec, _, _ = _spec(style, D)
    rope.table(spec, DEV)
    pool0 = pool.clone()
    prog = ops.Program()
    with prog.record():
        ops.wo_gemm(x, w, ws, out=qkv)
        rope.rope_append(spec, qkv, pool, pl, seq, Hq, q_out=q, qk_norm=(qg, kg, EPS))
    assert prog.num_ops == 1, "only the GEMM runs in the persistent kernel"
    prog.launch()
    torch.cuda.synchronize()
    pool_ref = pool0.clone()
    q_ref = _composition(spec, False, None, qkv, qg, kg, pool_ref, pl, seq, Hq, Hkv, D, 1)
    torch.cuda.synchronize()
    assert torch.equal(q, q_ref) and torch.equal(pool, pool_ref)
