"""GPU tests (H100) of speculative-token verification: paged attention at 17..64 query rows per (sequence, kv head), the
multi-token RoPE + K/V append, the draft verifier, and the verification step of DecodeStep against an op-by-op oracle."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests.step_oracle import TINY31, check_logits, check_step  # noqa: E402
from tests.verify_oracle import chain_verify_np  # noqa: E402

DEV = torch.device("cuda")
TILES = "B200_ATTN_TILES_PER_SPLIT"

# name, head_dim, B, q_len, Hq, Hkv, page, lens (cached before the q_len new tokens), dtype, env
ROWS = [
    ("g8 x q_len 4 p64", 128, 3, 4, 16, 2, 64, [10, 64, 300], torch.float16, None),
    ("g8 x q_len 8 p16 bf16", 128, 2, 8, 8, 1, 16, [5, 130], torch.bfloat16, None),
    ("g4 x q_len 16 d64 p32 cluster merge", 64, 2, 16, 8, 2, 32, [40, 700], torch.float16, {TILES: 2}),
    ("g16 x q_len 4 d256 p128", 256, 2, 4, 32, 2, 128, [127, 300], torch.float16, None),
    ("g16 x q_len 4 bf16 workspace merge", 128, 2, 4, 16, 1, 32, [900, 17], torch.bfloat16, {TILES: 1}),
    ("mqa g32 p64 workspace merge bf16", 128, 2, 1, 32, 1, 64, [900, 70], torch.bfloat16, {TILES: 1}),
    ("mqa g64 d256 p32 cluster merge", 256, 2, 1, 64, 1, 32, [500, 65], torch.float16, {TILES: 2}),
    ("mqa g64 d64 p16 bf16", 64, 3, 1, 64, 1, 16, [0, 15, 200], torch.bfloat16, None),
    ("g7 x q_len 3 p16", 128, 3, 3, 14, 2, 16, [0, 17, 200], torch.float16, None),
    ("g8 x q_len 8 d64 bf16 workspace merge", 64, 2, 8, 16, 2, 64, [900, 3], torch.bfloat16, {TILES: 1}),
]


def _attn_multi_vs_oracle(name, D, B, q_len, Hq, Hkv, T, lens, dtype, env, seed=5):
    with probe.env_set(env):
        is_bf16 = dtype == torch.bfloat16
        total = [L + q_len for L in lens]
        _, pool, block_ids, _ = probe.make_attn_case(B, Hq, Hkv, T, total, dtype, seed=seed, D=D)
        q = torch.randn(B, q_len, Hq, D, generator=torch.Generator().manual_seed(9)).to(dtype)
        seq = torch.tensor(lens, dtype=torch.int32)
        max_len = max(total)
        ws = ops.attn_workspace(B * q_len, Hq, Hkv, max_len, DEV)
        buf, out = probe.guarded_empty((B, q_len, Hq * D), dtype)
        ops.paged_decode_attn_multi(q.to(DEV), pool.to(DEV), ops.convert_block_table(block_ids.to(DEV)), seq.to(DEV), max_len, ws,
                                    out=out)
        torch.cuda.synchronize()
        probe.RESULTS.clear()
        f64, E = orc.paged_decode_attn_np(q.float().numpy(), pool.float().numpy(), block_ids.numpy(), seq.numpy(), T, with_abs=True)
        ok, info = probe.budget_info(out, f64, E, is_bf16)
        probe.report(name + " [kernel vs float64, error budget]", ok, info)
        probe.report_bands(name, buf)
        sem_clean = int(ws[: B * Hkv * 4].view(torch.int32).abs().sum().item()) == 0
        probe.report(name + " [semaphores reset]", sem_clean)
        bad = [n for n, ok in probe.RESULTS if not ok]
        assert not bad, bad
        bits = lambda t: t.contiguous().view(torch.int16).numpy().view(np.uint16)
        pl_np = orc.convert_block_table(block_ids.numpy())
        tol = 2e-2 if is_bf16 else 1e-2
        for j in range(q_len):
            exp = orc.from_bits(orc.paged_decode_attn(bits(q[:, j]), bits(pool), pl_np, (seq + j).numpy(), Hq, Hkv, D, T,
                                                      is_bf16=is_bf16), is_bf16)
            np.testing.assert_allclose(out[:, j].float().cpu().numpy(), exp, rtol=tol, atol=tol, err_msg=f"query token {j}")


@pytest.mark.parametrize("case", ROWS, ids=[c[0] for c in ROWS])
def test_attention_with_17_to_64_query_rows_vs_oracle(case):
    _attn_multi_vs_oracle(*case)


@pytest.mark.parametrize("case", ROWS, ids=[c[0] for c in ROWS])
def test_attention_with_17_to_64_query_rows_reads_exactly_the_visible_positions(case):
    name, D, B, q_len, Hq, Hkv, T, lens, dtype, env = case
    probe.RESULTS.clear()
    probe.attn_position_probes(name, B, Hq, Hkv, T, lens, dtype, env, D=D, q_len=q_len)
    bad = [n for n, ok in probe.RESULTS if not ok]
    assert probe.RESULTS and not bad, bad


def test_attention_64_rows_full_size_vs_oracle():
    """Qwen2-72B / Llama-3-70B group 8 with 7 drafts: Hq 64, Hkv 8, B 32, S 2048, q_len 8 (64 rows per kv head)."""
    _attn_multi_vs_oracle("Hq64 Hkv8 B32 S2048 q_len 8", 128, 32, 8, 64, 8, 64, [2048 - 8] * 32, torch.float16, None, seed=42)


ROPE = [("d128 p16 fp16", 128, 3, 4, 8, 2, 16, [0, 14, 100], torch.float16),
        ("d128 p64 bf16 q_len 8", 128, 2, 8, 16, 2, 64, [60, 500], torch.bfloat16),
        ("d64 p32 q_len 3", 64, 4, 3, 4, 4, 32, [31, 1, 64, 90], torch.float16)]


@pytest.mark.parametrize("case", ROPE, ids=[c[0] for c in ROPE])
def test_rope_append_multi_equals_single_token_appends(case):
    name, D, B, q_len, Hq, Hkv, T, lens, dtype = case
    g = torch.Generator(device=DEV).manual_seed(7)
    M = max(-(-(L + q_len) // T) for L in lens)
    P = B * M + 1
    pool1 = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    pool2 = pool1.clone()
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    pl = ops.convert_block_table((torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1).reshape(B, M))
    seq = torch.tensor(lens, dtype=torch.int32, device=DEV)
    q = ops.rope_append(qkv, pool1, pl, seq, Hq, 500000.0, q_len=q_len).view(B, q_len, -1)
    rows = qkv.view(B, q_len, -1)
    for j in range(q_len):
        qj = ops.rope_append(rows[:, j].contiguous(), pool2, pl, seq + j, Hq, 500000.0)
        assert torch.equal(q[:, j], qj), f"q of token {j} differs"
    torch.cuda.synchronize()
    assert torch.equal(pool1, pool2), "cache contents differ"


# ---------------------------------------------------------------------------------------------------- verifier
V_FULL = 128256


def check_verify(got, expected, u):
    """A verifier's outputs `got` (out_tokens, accepted[, accepted_path]) against verify_np's `expected`, u [B] the draw's
    uniforms. Accept decisions and the path exact; a drawn token exact unless u * total lies within 1e-6 * total of a CDF
    boundary of the mass the draw used. There the kernel's fp32 scan may pick another token with mass, whose CDF interval must
    then come within 1e-6 * total of u * total (in a tail of tiny probabilities that can be a few tokens away, not only a
    neighbour)."""
    got = [x.cpu().numpy() for x in got]
    exp, acc_exp, path_exp, masses = expected
    u = np.asarray(u, np.float64)
    np.testing.assert_array_equal(got[1], acc_exp)
    if len(got) > 2:
        np.testing.assert_array_equal(got[2], path_exp)
    got = got[0]
    for b in range(got.shape[0]):
        a = acc_exp[b]
        np.testing.assert_array_equal(got[b, :a], exp[b, :a])
        assert (got[b, a + 1:] == -1).all()
        if got[b, a] == exp[b, a]:
            continue
        m = masses[b].astype(np.float64)
        idx = np.nonzero(m > 0)[0]
        c = np.cumsum(m[idx])
        total, t = c[-1], u[b] * c[-1]
        tol = 1e-6 * total
        near = np.abs(np.concatenate([[0.0], c]) - t).min() <= tol
        k = int(np.searchsorted(idx, got[b, a]))
        assert near and k < idx.size and idx[k] == got[b, a], (b, a, got[b, a], exp[b, a])
        lo, hi = (c[k - 1] if k else 0.0), c[k]                           # the drawn token's CDF interval
        assert lo - tol <= t <= hi + tol, (b, a, got[b, a], exp[b, a], lo, hi, t, total)


@pytest.mark.parametrize("n", range(1, 8))
def test_spec_verify_greedy_vs_oracle(n):
    rng = np.random.default_rng(n)
    B = 32
    ids = rng.integers(0, V_FULL, (B, n + 1)).astype(np.int32)
    keep = rng.random((B, n)) < 0.8
    drafts = np.where(keep, ids[:, :n], rng.integers(0, V_FULL, (B, n))).astype(np.int32)
    out, acc = ops.spec_verify(torch.from_numpy(drafts).to(DEV), target_ids=torch.from_numpy(ids).to(DEV))
    eo, ea = chain_verify_np(drafts, target_ids=ids)[:2]
    np.testing.assert_array_equal(acc.cpu().numpy(), ea)
    np.testing.assert_array_equal(out.cpu().numpy(), eo)


def _probs(rng, shape, temp):
    x = torch.from_numpy(rng.standard_normal(shape).astype(np.float32)) / temp
    return torch.softmax(x, dim=-1).numpy()


@pytest.mark.parametrize("with_draft_probs", [True, False], ids=["draft probs", "deterministic drafts"])
@pytest.mark.parametrize("n", range(1, 8))
def test_spec_verify_sampling_vs_oracle(n, with_draft_probs):
    rng = np.random.default_rng(100 + n)
    B = 32
    t = _probs(rng, (B, n + 1, V_FULL), 0.25)
    dp = (0.5 * t[:, :n] + 0.5 * _probs(rng, (B, n, V_FULL), 0.25)).astype(np.float32) if with_draft_probs else None
    src = dp if with_draft_probs else t[:, :n]
    drafts = np.array([[rng.choice(V_FULL, p=src[b, i].astype(np.float64) / src[b, i].astype(np.float64).sum()) for i in range(n)]
                       for b in range(B)], np.int32)
    # edge rows: a mass-free target row, a draft of draft probability 0, a rejection whose residual has no mass
    t[0, 0] = 0.0
    if with_draft_probs:
        dp[1, 0, drafts[1, 0]] = 0.0
        dp[2, 0] = 2.0 * t[2, 0]
    else:
        t[2, 0] = 0.0
        t[2, 0, drafts[2, 0]] = 0.7
    u = rng.random((B, n + 1)).astype(np.float32)
    u[2, 0] = 0.9                                   # rejects row 2's first draft in both modes
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    got = ops.spec_verify(T(drafts), target_probs=T(t), draft_probs=T(dp), uniform=T(u))
    exp = chain_verify_np(drafts, target_probs=t, draft_probs=dp, uniform=u)
    check_verify(got, exp, u[:, n])
    eo, ea = exp[:2]
    got = got[0].cpu().numpy()
    assert ea[0] == 0 and eo[0, 0] == -1                   # mass-free row: rejected, nothing to draw
    assert ea[2] == 0 and got[2, 0] >= 0
    if with_draft_probs:
        assert ea[1] >= 1                                  # p = 0 < q: accepted whatever the uniform


# ---------------------------------------------------------------------------------------------------- decode step
STEP = [(q, n, "eager") for q in ("int4", "int8", "int8g", "f16") for n in (2, 4)] + \
       [("int4", 4, "graph"), ("int4", 4, "pdl"), ("f16", 2, "graph pdl"), ("int8g", 4, "graph")]


@pytest.mark.parametrize("case", STEP, ids=[f"{q} q_len {n} {m}" for q, n, m in STEP])
def test_verification_step_vs_oracle(case):
    quant, q_len, mode = case
    check_step(quant=quant, batch=3, ctx=40, mode=mode, q_len=q_len, dev=DEV)


def test_verification_step_is_not_a_program():
    model = DecodeStep(TINY, 2, 40, DEV, q_len=2)
    with pytest.raises(ValueError, match="program"):
        model.build_program()


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("cfg", [dataclasses.replace(TINY, quant="int4"), TINY31], ids=["int4", "llama31"])
def test_verification_step_accepts_the_tokens_plain_steps_produce(cfg, k):
    """k greedy single-token steps on one model, then one q_len = k + 1 step on an identical model with those tokens as drafts:
    row j's logits match plain step j, and wherever every plain step's top-2 margin is clear of the error, all k drafts are
    accepted and the emitted token is plain step k's. Everywhere, the verifier's decisions are those of the reference on the
    step's own greedy rows."""
    plain = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2)
    spec = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2, q_len=k + 1)
    plain.seq_lens_h.copy_(spec.seq_lens_h)
    plain.ids_h.copy_(spec.ids_h[:, 0])
    toks, logits = [plain.ids_h.clone()], []
    for _ in range(k + 1):
        plain.upload_inputs()
        plain.run()
        torch.cuda.synchronize()
        logits.append(plain.logits.float().cpu().numpy())
        toks.append(plain.next_ids.cpu())
        plain.ids_h.copy_(plain.next_ids.cpu())
        plain.seq_lens_h += 1
    spec.ids_h.copy_(torch.stack(toks[:k + 1], dim=1))
    spec.upload_inputs()
    spec.run()
    torch.cuda.synchronize()
    got = spec.logits.float().cpu().numpy().reshape(spec.B, k + 1, -1)
    exp = np.stack(logits, axis=1)
    err = check_logits(got, exp)
    srt = np.sort(exp, axis=-1)
    sure = ((srt[..., -1] - srt[..., -2]) > 2 * err + 1e-6).all(axis=1)
    assert sure.any(), "no sequence with a clear margin at every step"
    acc, out = spec.accepted.cpu().numpy(), spec.out_tokens.cpu().numpy()
    assert (acc[sure] == k).all(), acc
    np.testing.assert_array_equal(out[sure, k], toks[k + 1].numpy()[sure])
    np.testing.assert_array_equal(out[sure, :k], torch.stack(toks[1:k + 1], dim=1).numpy()[sure])
    eo, ea = chain_verify_np(spec.ids_h[:, 1:].numpy(), target_ids=spec.next_ids.view(spec.B, k + 1).cpu().numpy())[:2]
    np.testing.assert_array_equal(acc, ea)
