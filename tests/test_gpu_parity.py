"""GPU parity tests (run with -m gpu on an H100). Everything goes through the C ABI
(rtp_llm_b200.ops -> libb200_decode.so) and is compared with the CPU oracle on the same seeded inputs, with the golden
fixtures the reference's code produced -- at BASELINE.json's full sizes too (the OpenMP oracle finishes those in well under
a second per case); a deliberately naive GPU kernel (test-only library) is kept as a second opinion."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8, B200_FMT_INT8G  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402


def _run(fn, *a, **k):
    probe.RESULTS.clear()
    fn(*a, **k)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad


def test_native_library_is_the_path_that_runs():
    ops.device_check(0)
    n0 = ops.launch_count()
    ops.convert_block_table(torch.zeros(2, 4, dtype=torch.int32, device="cuda"))
    assert ops.launch_count() == n0 + 1


@pytest.mark.parametrize("name", ["attn_p16_gqa4", "attn_p64_gqa8", "attn_p32_mha"])
def test_attention_matches_reference_golden(golden_dir, name):
    """Fixtures produced by the reference's own torch oracle (oracle/make_golden.py); tolerance = the reference's
    rtol = atol = 1e-2 (base_attention_test.py:147-148)."""
    g = np.load(os.path.join(golden_dir, f"{name}.npz"))
    dev = torch.device("cuda")
    q = torch.from_numpy(g["q"]).to(dev)
    pool = torch.from_numpy(g["kv_pool"]).to(dev)
    bid = torch.from_numpy(g["block_ids"]).to(dev)
    seq = torch.from_numpy(g["sequence_lengths"]).to(dev)
    pl = ops.convert_block_table(bid)
    max_len = int(g["sequence_lengths"].max()) + 1
    ws = ops.attn_workspace(q.shape[0], int(g["head_num"]), int(g["kv_head_num"]), max_len, dev)
    out = ops.paged_decode_attn(q, pool, pl, seq, max_len, ws)
    torch.cuda.synchronize()
    np.testing.assert_allclose(out.float().cpu().numpy(), g["expect"], rtol=1e-2, atol=1e-2)


ATTN_CASES = [
    ("B1 len1", 1, 4, 1, 64, [1], torch.float16, None),
    ("len 10/64", 2, 8, 2, 64, [10, 64], torch.float16, None),                     # test_xqa.py:368-449 shapes
    ("len 65..513", 4, 8, 2, 64, [65, 128, 200, 513], torch.float16, None),
    ("page16", 4, 8, 2, 16, [10, 20, 65, 130], torch.float16, None),
    ("page32 mha", 3, 4, 4, 32, [64, 65, 1], torch.float16, None),
    ("page128 g8", 3, 16, 2, 128, [127, 129, 300], torch.float16, None),
    ("g16", 2, 16, 1, 64, [100, 257], torch.float16, None),
    ("bf16", 3, 8, 2, 64, [63, 64, 300], torch.bfloat16, None),
    ("split every tile", 3, 8, 2, 64, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("no split", 3, 8, 2, 64, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1000}),
    # 2..8 splits merge through a thread-block cluster (DSMEM); short sequences leave some CTAs of the cluster without tokens
    ("cluster merge 6 splits ragged", 3, 8, 2, 64, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}),
    ("cluster merge 8 splits g16", 2, 16, 1, 64, [500, 1], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("cluster merge 2 splits bf16 p16", 4, 8, 2, 16, [10, 20, 65, 128], torch.bfloat16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("cluster merge 3 splits mha p32", 3, 4, 4, 32, [64, 65, 190], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    # attention.py passes q_scale = 1 / q_scaling
    ("q_scale 0.5", 4, 8, 2, 64, [65, 128, 200, 513], torch.float16, None, dict(q_scale=0.5)),
    ("q_scale 1/1.3 bf16 cluster merge", 3, 8, 2, 64, [63, 64, 700], torch.bfloat16, {"B200_ATTN_TILES_PER_SPLIT": 2},
     dict(q_scale=1 / 1.3)),
    # callers pass a loose bound on the lengths, and the split plan follows the bound, not the lengths
    ("max_seq_len 4096", 3, 8, 2, 64, [100, 700, 1500], torch.float16, None, dict(max_len=4096)),
    ("max_seq_len 8192 lengths 1..70", 70, 8, 2, 64, list(range(1, 71)), torch.bfloat16, None, dict(max_len=8192)),
]


@pytest.mark.parametrize("case", ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def test_attention_vs_oracle(case):
    name, B, Hq, Hkv, T, lens, dtype, env, *kw = case
    _run(probe.attn_vs_oracle, name, B, Hq, Hkv, T, lens, dtype, env, **(kw[0] if kw else {}))


HEAD_DIMS = [
    ("d64 g4 ragged", 64, 4, 8, 2, 64, [1, 64, 65, 513], torch.float16, None),
    ("d64 mha p16 bf16", 64, 3, 4, 4, 16, [10, 20, 130], torch.bfloat16, None),
    ("d64 cluster splits", 64, 3, 8, 2, 64, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}),
    ("d64 workspace splits g16", 64, 2, 16, 1, 32, [900, 2], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("d256 g4 ragged", 256, 4, 8, 2, 64, [1, 64, 65, 513], torch.float16, None),
    ("d256 g8 p128 bf16", 256, 3, 16, 2, 128, [127, 129, 300], torch.bfloat16, None),
    ("d256 cluster splits", 256, 3, 8, 2, 64, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}),
    ("d256 workspace splits", 256, 2, 4, 1, 16, [600, 3], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
]


@pytest.mark.parametrize("case", HEAD_DIMS, ids=[c[0] for c in HEAD_DIMS])
def test_attention_head_dim_64_and_256_vs_oracle(case):
    """The head sizes XQA ships next to 128 (3rdparty/xqa/def.bzl:49-78): same kernel, templated on head_dim."""
    name, D, B, Hq, Hkv, T, lens, dtype, env = case
    _run(probe.attn_vs_oracle, name, B, Hq, Hkv, T, lens, dtype, env, D=D)


MULTI_Q = [
    ("q_len 4 g4", 3, 4, 8, 2, 64, [10, 64, 300], torch.float16, None),
    ("q_len 2 g8 p16 bf16", 3, 2, 16, 2, 16, [5, 17, 130], torch.bfloat16, None),
    ("q_len 11 mha", 2, 11, 2, 2, 32, [40, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}),
    ("q_len 3 g4 workspace splits", 2, 3, 4, 1, 64, [900, 70], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("q_len 16 g1 crossing a tile", 1, 16, 1, 1, 64, [70], torch.float16, None),
]


@pytest.mark.parametrize("case", MULTI_Q, ids=[c[0] for c in MULTI_Q])
def test_attention_with_several_query_tokens_vs_oracle(case):
    """q_len speculative tokens per sequence (XQA max_q_len / trtllm-gen q_len_per_req): query j must equal a plain decode
    attention over the first sequence_lengths + j + 1 positions. Checked against the float64 reference within the error
    budget, with the C oracle (one call per j) as a second opinion at 1e-2 (bf16: 2e-2)."""
    name, B, q_len, Hq, Hkv, T, lens, dtype, env = case          # lens = tokens cached BEFORE the q_len new ones
    with probe.env_set(env):
        dev = torch.device("cuda")
        is_bf16 = dtype == torch.bfloat16
        total = [L + q_len for L in lens]
        _, pool, block_ids, _ = probe.make_attn_case(B, Hq, Hkv, T, total, dtype, seed=5)
        g = torch.Generator().manual_seed(9)
        q = torch.randn(B, q_len, Hq, 128, generator=g).to(dtype)
        seq = torch.tensor(lens, dtype=torch.int32)
        pl = ops.convert_block_table(block_ids.to(dev))
        max_len = max(total)
        ws = ops.attn_workspace(B * q_len, Hq, Hkv, max_len, dev)
        buf, out = probe.guarded_empty((B, q_len, Hq * 128), dtype)
        ops.paged_decode_attn_multi(q.to(dev), pool.to(dev), pl, seq.to(dev), max_len, ws, out=out)
        torch.cuda.synchronize()
        probe.RESULTS.clear()
        f64, E = orc.paged_decode_attn_np(q.float().numpy(), pool.float().numpy(), block_ids.numpy(), seq.numpy(), T,
                                          with_abs=True)
        ok, info = probe.budget_info(out, f64, E, is_bf16)
        probe.report(name + " [kernel vs float64, error budget]", ok, info)
        probe.report_bands(name, buf)
        bad = [n for n, ok in probe.RESULTS if not ok]
        assert not bad, bad
        bits = lambda t: t.contiguous().view(torch.int16).numpy().view(np.uint16)
        pl_np = orc.convert_block_table(block_ids.numpy())
        tol = 2e-2 if is_bf16 else 1e-2
        for j in range(q_len):
            exp = orc.from_bits(orc.paged_decode_attn(bits(q[:, j]), bits(pool), pl_np, (seq + j).numpy(), Hq, Hkv, 128, T,
                                                      is_bf16=is_bf16), is_bf16)
            np.testing.assert_allclose(out[:, j].float().cpu().numpy(), exp, rtol=tol, atol=tol, err_msg=f"query token {j}")


@pytest.mark.parametrize("cfg", [("Llama-3-8B B32 S2048", 32, 32, 8, 64, 2048, False, torch.float16),
                                 ("Llama-3-8B B32 S2048 ragged", 32, 32, 8, 64, 2048, True, torch.float16),
                                 ("Llama-3-8B B32 S2048 bf16", 32, 32, 8, 64, 2048, False, torch.bfloat16),
                                 ("Qwen2-72B TP8 B16 S8192", 16, 8, 1, 64, 8192, False, torch.float16),
                                 ("Qwen2-72B TP8 B16 S8192 bf16", 16, 8, 1, 64, 8192, False, torch.bfloat16)],
                         ids=lambda c: c[0])
def test_attention_full_size_vs_oracle(cfg):
    name, B, Hq, Hkv, T, S, ragged, dtype = cfg
    _run(probe.attn_vs_ref_big, name, B, Hq, Hkv, T, S, dtype, ragged)


POSITION_PROBES = [
    # name, head_dim, B, q_len, Hq, Hkv, page, lens (cached before the new tokens), dtype, env, max_seq_len
    ("p16 g4", 128, 4, 1, 8, 2, 16, [0, 15, 16, 130], torch.float16, None, None),
    ("p32 mha d64 bf16", 64, 3, 1, 4, 4, 32, [31, 32, 200], torch.bfloat16, None, None),
    ("p64 g8 d256", 256, 3, 1, 16, 2, 64, [63, 64, 513], torch.float16, None, None),
    ("p128 g16 bf16", 128, 3, 1, 16, 1, 128, [127, 128, 300], torch.bfloat16, None, None),
    ("cluster merge 8 splits g4", 128, 2, 1, 8, 2, 64, [500, 65], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}, None),
    ("cluster merge 4 splits d64 p16 bf16", 64, 3, 1, 8, 2, 16, [130, 400, 7], torch.bfloat16,
     {"B200_ATTN_TILES_PER_SPLIT": 2}, None),
    ("workspace merge g8 p32 bf16", 128, 2, 1, 16, 2, 32, [900, 70], torch.bfloat16, {"B200_ATTN_TILES_PER_SPLIT": 1}, None),
    ("workspace merge d256 g4 p16", 256, 2, 1, 4, 1, 16, [600, 3], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}, None),
    ("max_seq_len 8192 lengths 1..70", 128, 70, 1, 8, 2, 64, list(range(0, 70)), torch.float16, None, 8192),
    ("q_len 4 g4 p64", 128, 3, 4, 8, 2, 64, [10, 60, 300], torch.float16, None, None),
    ("q_len 2 g8 p16 bf16 workspace merge", 128, 2, 2, 16, 2, 16, [900, 17], torch.bfloat16,
     {"B200_ATTN_TILES_PER_SPLIT": 1}, None),
    ("q_len 16 mha p32 cluster merge", 128, 2, 16, 2, 2, 32, [60, 300], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}, None),
]


@pytest.mark.parametrize("case", POSITION_PROBES, ids=[c[0] for c in POSITION_PROBES])
def test_attention_reads_exactly_the_visible_positions(case):
    """Exact probes (uniform scores, dominant key): an output off by one token, page, kv head or batch row fails at any
    sequence length, where a tolerance check would lose it in the average."""
    name, D, B, q_len, Hq, Hkv, T, lens, dtype, env, max_len = case
    _run(probe.attn_position_probes, name, B, Hq, Hkv, T, lens, dtype, env, D=D, q_len=q_len, max_len=max_len)


ROPE_FUSED = [
    ("g4 p64 ragged", 4, 8, 2, 64, [1, 64, 65, 513], torch.float16, None),
    ("g8 p16 bf16", 3, 16, 2, 16, [10, 16, 130], torch.bfloat16, None),
    ("mha p32 cluster splits", 3, 4, 4, 32, [63, 64, 700], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 2}),
    ("g16 workspace splits", 2, 16, 1, 64, [900, 2], torch.float16, {"B200_ATTN_TILES_PER_SPLIT": 1}),
    ("Llama B32 S2048", 32, 32, 8, 64, [2048] * 32, torch.float16, None),
]


@pytest.mark.parametrize("case", ROPE_FUSED, ids=[c[0] for c in ROPE_FUSED])
def test_attention_with_fused_rope_is_bit_identical_to_rope_then_attention(case):
    """b200_paged_decode_attn_rope == b200_rope_append followed by b200_paged_decode_attn, bit for bit (output and cache)."""
    name, B, Hq, Hkv, T, lens, dtype, env = case
    old = {}
    for k, v in (env or {}).items():
        old[k] = os.environ.get(k)
        os.environ[k] = str(v)
    try:
        dev = torch.device("cuda")
        g = torch.Generator(device=dev).manual_seed(len(name))
        D = 128
        M = max((L + T - 1) // T for L in lens)
        P = B * M + 1
        pool1 = torch.randn(P, 2, Hkv, T, D, generator=g, device=dev).to(dtype)
        pool2 = pool1.clone()
        qkv = torch.randn(B, (Hq + 2 * Hkv) * D, generator=g, device=dev).to(dtype)
        bid = (torch.randperm(P - 1, generator=g, device=dev).to(torch.int32) + 1).reshape(B, M)
        pl = ops.convert_block_table(bid)
        seq = torch.tensor([L - 1 for L in lens], dtype=torch.int32, device=dev)
        max_len = max(lens)
        ws = ops.attn_workspace(B, Hq, Hkv, max_len, dev)
        q = ops.rope_append(qkv, pool1, pl, seq, Hq, 500000.0)
        out1 = ops.paged_decode_attn(q, pool1, pl, seq, max_len, ws)
        out2 = ops.paged_decode_attn_rope(qkv, pool2, pl, seq, Hq, max_len, 500000.0, ws)
        torch.cuda.synchronize()
        assert torch.equal(pool1, pool2), "appended K/V differ"
        assert torch.equal(out1, out2), f"attention output differs: max {(out1.float() - out2.float()).abs().max().item()}"
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


GEMM_SMALL = [
    ("onehot", 16, 128, 128, dict(simple=True, onehot=True)),
    ("B16 K256 N256", 16, 256, 256, {}),
    ("B5 K512 N384 bias", 5, 512, 384, dict(bias=True)),
    ("splitk4", 32, 1024, 256, dict(env={"B200_GEMM_SPLITK": 4})),
    ("ragged N bpad64", 33, 512, 200, {}),
    ("bpad128", 100, 512, 256, {}),
    ("bf16", 8, 256, 256, dict(dtype=torch.bfloat16)),
    # uneven cluster split-K (runs 3, 3, 2), and 8 splits forced on 3 k-blocks (clamped to 3 single-block runs)
    ("splitk3 bias", 19, 1024, 384, dict(env={"B200_GEMM_SPLITK": 3}, bias=True)),
    ("splitk8 clamped K384", 32, 384, 256, dict(env={"B200_GEMM_SPLITK": 8})),
    # one split over 25 k-blocks: an odd run that wraps every stage ring more than twice, at every batch pad
    ("ring wrap B1", 1, 3200, 256, dict(env={"B200_GEMM_SPLITK": 1})),
    ("ring wrap B17", 17, 3200, 256, dict(env={"B200_GEMM_SPLITK": 1})),
    ("ring wrap B64", 64, 3200, 256, dict(env={"B200_GEMM_SPLITK": 1})),
    ("ring wrap B128", 128, 3200, 256, dict(env={"B200_GEMM_SPLITK": 1})),
    ("ring wrap B17 bf16", 17, 3200, 256, dict(env={"B200_GEMM_SPLITK": 1}, dtype=torch.bfloat16)),
    # batch pad edges (16 | 17, 64 | 65), single-request decode, the largest batch, and a last tile of 8 features
    ("B1", 1, 512, 256, {}),
    ("B16", 16, 512, 256, {}),
    ("B17", 17, 512, 256, {}),
    ("B64", 64, 512, 256, {}),
    ("B65", 65, 512, 256, {}),
    ("B128", 128, 512, 256, {}),
    ("N136", 17, 512, 136, {}),
]


@pytest.mark.parametrize("fmt", [B200_FMT_F16, B200_FMT_INT8, B200_FMT_INT4, B200_FMT_INT8G], ids=["f16", "int8", "int4", "int8g"])
@pytest.mark.parametrize("case", GEMM_SMALL, ids=[c[0] for c in GEMM_SMALL])
def test_gemm_vs_oracle(fmt, case):
    """Primary check: the float64 reference within oracle.gemm_error_budget, with the correctly rounded fractions above
    their thresholds (the reference has no weight-only GEMM kernel to pin against, SURVEY 8c). Second opinions at
    |d| <= 1e-2*|y| + 1e-2 for FP16/INT8 weights, 2e-2 for INT4: the C oracle and the naive GPU kernel."""
    name, B, K, N, kw = case
    _run(probe.gemm_case, f"{name}", fmt, B, K, N, **kw)


@pytest.mark.parametrize("cfg", [("int4 Llama qkv B32", B200_FMT_INT4, 32, 4096, 6144),
                                 ("int4 Llama w2 B32", B200_FMT_INT4, 32, 14336, 4096),
                                 ("int4 Llama w13 B64", B200_FMT_INT4, 64, 4096, 28672),
                                 ("int8 Llama o B32", B200_FMT_INT8, 32, 4096, 4096),
                                 ("int8 group-wise Llama qkv B32", B200_FMT_INT8G, 32, 4096, 6144),
                                 ("f16 lm_head slice B32", B200_FMT_F16, 32, 4096, 16032)], ids=lambda c: c[0])
def test_gemm_full_size_vs_oracle(cfg):
    """BASELINE shapes: checked against the CPU oracle (and, as a second opinion, the naive GPU kernel)."""
    name, fmt, B, K, N = cfg
    _run(probe.gemm_case, name, fmt, B, K, N, big=True)


PERSISTENT = [
    ("uniform split", B200_FMT_INT4, 32, 1024, 256, {}),
    ("uniform split bias int8", B200_FMT_INT8, 19, 1024, 384, dict(bias=True)),
    ("2-way split bf16", B200_FMT_INT4, 8, 256, 256, dict(dtype=torch.bfloat16)),
    ("ragged N bpad64", B200_FMT_INT4, 33, 512, 200, {}),
    ("Llama w2 B32", B200_FMT_INT4, 32, 14336, 4096, dict(big=True)),
    ("16 contributors", B200_FMT_INT4, 32, 2048, 128, {}),
    ("whole tiles", B200_FMT_INT4, 8, 128, 256, {}),
    ("several tiles per CTA int8", B200_FMT_INT8, 8, 256, 76800, {}),
    ("workspace for B16 forces longer runs", B200_FMT_INT4, 40, 1024, 256, dict(ws_batch=16)),
]


@pytest.mark.parametrize("case", PERSISTENT, ids=[c[0] for c in PERSISTENT])
def test_gemm_persistent_kernel_standalone(case):
    """The persistent kernel of the decode programs (csrc/decode_program.cuh) run as a one-op program: split tiles merged
    by all their contributors, and whole tiles stored directly. The probe checks that the GEMM was recorded as an op of the
    persistent kernel, not replayed through the cluster kernel.

    The last four shapes reach the branches of the run-length plan (sk_plan in c_api.cu) for any grid of 16 to 2 x 132
    CTAs: one tile of 16 k-blocks is split 16 ways (the merge loop over contributors 8..15); one k-block per tile gives
    whole tiles; 600 tiles of 2 k-blocks give each CTA several whole tiles, and at 264 CTAs leave 64 of them idle; a
    workspace sized for batch 16 cannot hold the 8 partials of batch pad 64, so the plan falls back to 2 runs of 4."""
    name, fmt, B, K, N, kw = case
    _run(probe.gemm_case, name, fmt, B, K, N, program=True, **kw)
    _run(probe.gemm_silu_case, name + " silu", fmt, 7, 512, 192, program=True)


@pytest.mark.parametrize("fmt", [B200_FMT_F16, B200_FMT_INT8, B200_FMT_INT4, B200_FMT_INT8G], ids=["f16", "int8", "int4", "int8g"])
def test_gemm_fused_silu_mul_vs_oracle(fmt):
    _run(probe.gemm_silu_case, "silu direct", fmt, 7, 256, 192)
    _run(probe.gemm_silu_case, "silu cluster split", fmt, 32, 1024, 128, env={"B200_GEMM_SPLITK": 4})


def test_gemm_is_linear_in_x():
    """Size-independent property at a BASELINE shape: Y(a*x1 + x2) == a*Y(x1) + Y(x2) within fp16 rounding."""
    dev = torch.device("cuda")
    K, N, B = 4096, 4096, 32
    qp, s, zs = probe.make_w4(K, N)
    w = ops.pack_w4(torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dev), torch.from_numpy(zs).to(dev))
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    g = torch.Generator(device=dev).manual_seed(0)
    x1 = torch.randn(B, K, generator=g, device=dev).half()
    x2 = torch.randn(B, K, generator=g, device=dev).half()
    y1 = ops.wo_gemm(x1, w, ws).float()
    y2 = ops.wo_gemm(x2, w, ws).float()
    y3 = ops.wo_gemm((2 * x1 + x2), w, ws).float()
    torch.testing.assert_close(y3, 2 * y1 + y2, rtol=2e-2, atol=2e-2 * float(y3.abs().mean()) + 2e-2)


def test_glue_ops_and_indexing_vs_oracle():
    _run(probe.glue_cases)
