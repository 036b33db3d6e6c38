"""The glue ops' float64 references and error budgets (oracle.rmsnorm_np / norm_error_budget, rope_np / rope_error_budget,
silu_mul_budget with exact inputs, and the rounded-fraction thresholds), without a GPU: the fp32 C oracles, written
independently of the CUDA code, pass every check at the GPU tests' shapes, and each subtly wrong numpy kernel fails one."""
import numpy as np
import pytest

from oracle import oracle as orc

BASE = dict(style=1, dim=128, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=2048, extrapolation_factor=1.0, mscale=1.0)


def bits(v, is_bf16):
    return orc.f64_to_bits(v, is_bf16)


def violations(got, ref, budget, is_bf16):
    """(outputs outside the budget -- a NaN counts --, worst err/budget); got: T values or uint16 bits"""
    got = np.asarray(got)
    got = orc.from_bits(got, is_bf16) if got.dtype == np.uint16 else got
    r = np.abs(got.astype(np.float64) - ref) / budget
    return int((~(r <= 1.0)).sum()), float(np.nanmax(np.where(np.isfinite(r), r, np.inf)))


# ---------------------------------------------------------------------------------------------- RMSNorm
def norm_case(rng, rows, hidden, is_bf16, small_every=3):
    """x, residual, gamma as T values: N(0, 1) rows, every `small_every`-th row scaled to an RMS near 1e-3 (eps matters)."""
    scale = np.where(np.arange(rows) % small_every == 1, 1e-3, 1.0)[:, None]
    x = orc.round_t(rng.standard_normal((rows, hidden)) * scale, is_bf16)
    r = orc.round_t(rng.standard_normal((rows, hidden)) * scale, is_bf16)
    g = orc.round_t(rng.uniform(0.5, 1.5, hidden), is_bf16)
    return x, r, g


def norm_checks(y, ref, A, hidden, is_bf16, threads=128):
    n, worst = violations(y, ref, orc.norm_error_budget(ref, A, orc.norm_chain(hidden, threads), is_bf16), is_bf16)
    eq, one = orc.gemm_rounded_fractions(y, ref, is_bf16)
    return n, worst, (eq, one), eq >= orc.NORM_MIN_ROUNDED and one >= orc.NORM_MIN_WITHIN_ONE


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("hidden,rows,eps,with_res", [(8, 1, 1e-5, True), (1000, 33, 1e-6, True), (4096, 16, 1e-5, False),
                                                      (8192, 8, 1e-6, True), (12288, 4, 1e-5, True)])
def test_c_oracle_norm_within_budget(is_bf16, hidden, rows, eps, with_res):
    rng = np.random.default_rng(hidden + rows)
    x, r, g = norm_case(rng, rows, hidden, is_bf16)
    r = r if with_res else None
    y, res = orc.add_rmsnorm(bits(x, is_bf16), None if r is None else bits(r, is_bf16), bits(g, is_bf16), eps, is_bf16)
    ref, s, A = orc.rmsnorm_np(x, r, g, eps)
    n, worst, fr, ok_frac = norm_checks(y, ref, A, hidden, is_bf16)
    print(f"C oracle add_rmsnorm hidden {hidden}: worst err/budget {worst:.3f}, rounded / within one step {fr}")
    assert n == 0 and worst < 1.0 and ok_frac, (n, worst, fr)
    if r is not None:
        assert np.array_equal(res, bits(s, is_bf16))


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("D,with_bias", [(64, False), (128, True), (256, True)])
def test_c_oracle_qk_rmsnorm_within_budget(is_bf16, D, with_bias):
    rng = np.random.default_rng(D)
    R, Hq, Hkv = 7, 4, 2
    x = orc.round_t(rng.standard_normal((R, (Hq + 2 * Hkv) * D)), is_bf16)
    qg, kg = (orc.round_t(rng.uniform(0.5, 1.5, D), is_bf16) for _ in range(2))
    qb, kb = (orc.round_t(0.1 * rng.standard_normal(D), is_bf16) for _ in range(2)) if with_bias else (None, None)
    got = orc.from_bits(orc.qk_rmsnorm(bits(x, is_bf16), bits(qg, is_bf16), bits(kg, is_bf16), Hq, Hkv, D, 1e-6,
                                       None if qb is None else bits(qb, is_bf16), None if kb is None else bits(kb, is_bf16), is_bf16),
                        is_bf16).reshape(R, -1, D).astype(np.float64)
    h = x.reshape(R, -1, D)
    yq, _, Aq = orc.rmsnorm_np(h[:, :Hq], None, qg, 1e-6, qb)
    yk, _, Ak = orc.rmsnorm_np(h[:, Hq:Hq + Hkv], None, kg, 1e-6, kb)
    ref, A = np.concatenate([yq, yk], 1), np.concatenate([Aq, Ak], 1)
    n, worst = violations(got[:, :Hq + Hkv], ref, orc.norm_error_budget(ref, A, D // 32 + 5, is_bf16), is_bf16)
    eq, one = orc.gemm_rounded_fractions(bits(got[:, :Hq + Hkv], is_bf16), ref, is_bf16)
    print(f"C oracle qk_rmsnorm D {D}: worst err/budget {worst:.3f}, rounded / within one step {(eq, one)}")
    assert n == 0 and eq >= orc.NORM_MIN_ROUNDED and one >= orc.NORM_MIN_WITHIN_ONE
    assert np.array_equal(got[:, Hq + Hkv:], h[:, Hq + Hkv:])


NORM_MUTANTS = ["y rounded twice", "s rounded to T before the variance", "eps outside the square root",
                "mean over a padded width"]


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("name", NORM_MUTANTS)
def test_norm_mutant_is_rejected(is_bf16, name):
    hidden, eps = 1000, 1e-5                       # 1000: a width the kernels' 8-wide vectors pad to 1024
    rng = np.random.default_rng(5)
    x, r, g = norm_case(rng, 24, hidden, is_bf16)
    ref, s, A = orc.rmsnorm_np(x, r, g, eps)
    ms = lambda v: np.mean(v * v, -1, keepdims=True)
    if name == "y rounded twice":
        y = orc.round_t(orc.round_t(s / np.sqrt(ms(s) + eps), is_bf16) * g, is_bf16)
    elif name == "s rounded to T before the variance":
        sr = orc.round_t(s, is_bf16)
        y = orc.round_t(sr * g / np.sqrt(ms(sr) + eps), is_bf16)
    elif name == "eps outside the square root":
        y = orc.round_t(s * g / (np.sqrt(ms(s)) + eps), is_bf16)
    else:
        y = orc.round_t(s * g / np.sqrt((s * s).sum(-1, keepdims=True) / 1024 + eps), is_bf16)
    n, worst, fr, ok_frac = norm_checks(y, ref, A, hidden, is_bf16)
    print(f"norm mutant '{name}': {n} outputs outside the budget (worst {worst:.3g}), rounded / within one step {fr}")
    assert n > 0 or not ok_frac


# ---------------------------------------------------------------------------------------------- SiLU*mul
@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
def test_c_oracle_silu_mul_within_budget(is_bf16):
    rng = np.random.default_rng(3)
    inter = 1024
    gu = rng.standard_normal((16, 2 * inter)) * 3
    gu[0, :12] = [20, -20, 88, -88, 100, -100, 0, 1e-3, -1e-3, 5, -5, 10]
    gu = orc.round_t(gu, is_bf16)
    y = orc.silu_and_mul(bits(gu, is_bf16), is_bf16)
    g, u = gu[:, :inter], gu[:, inter:]
    ref = orc.silu_mul_np(g, u)
    n, worst = violations(orc.from_bits(y, is_bf16), ref, orc.silu_mul_budget(g, 0.0, u, 0.0, 128, 1, is_bf16), is_bf16)
    eq, one = orc.gemm_rounded_fractions(y, ref, is_bf16)
    print(f"C oracle silu_and_mul: worst err/budget {worst:.3f}, rounded / within one step {(eq, one)}")
    assert n == 0 and eq >= orc.SILU_MIN_ROUNDED and one >= orc.SILU_MIN_WITHIN_ONE


# ---------------------------------------------------------------------------------------------- RoPE
POSITIONS = np.array([0, 1, 15, 16, 63, 64, 2049, 4097, 8191, 32767, 65535, 131071], np.int32)


def plain_case(is_bf16, D=128, Hq=8, Hkv=2, T=16, base=1e6, positions=POSITIONS, seed=0):
    rng = np.random.default_rng(seed)
    B = len(positions)
    qkv = orc.round_t(rng.standard_normal((B, (Hq + 2 * Hkv) * D)), is_bf16)
    return qkv, dict(Hq=Hq, Hkv=Hkv, D=D, T=T, base=base, pos=np.asarray(positions, np.int32))


def c_rope_plain(qkv, c, is_bf16):
    """The C oracle's q_out and new K / V rows, [B, Hq + 2 Hkv, D] values."""
    B, T = qkv.shape[0], c["T"]
    M = int(c["pos"].max()) // T + 1
    block_ids = np.zeros((B, M), np.int32)
    block_ids[np.arange(B), c["pos"] // T] = 1 + np.arange(B)
    pool = np.zeros((1 + B, 2, c["Hkv"], T, c["D"]), np.uint16)
    q, pool = orc.rope_append(bits(qkv, is_bf16), pool, orc.convert_block_table(block_ids), c["pos"], c["Hq"], c["Hkv"], c["D"], T,
                              c["base"], is_bf16)
    kv = pool[1 + np.arange(B), :, :, c["pos"] % T]                   # [B, 2, Hkv, D]
    out = np.concatenate([q.reshape(B, c["Hq"], c["D"]), kv[:, 0], kv[:, 1]], 1)
    return orc.from_bits(out, is_bf16).astype(np.float64)


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("D,base", [(64, 10000.0), (128, 500000.0), (256, 1e6)])
def test_c_oracle_rope_append_within_budget(is_bf16, D, base):
    qkv, c = plain_case(is_bf16, D=D, base=base)
    got = c_rope_plain(qkv, c, is_bf16)
    ref, R, dA = orc.rope_np(qkv, c["Hq"], c["Hkv"], D, c["pos"], base=base, is_bf16=is_bf16)
    n, worst = violations(got, ref, orc.rope_error_budget(ref, R, dA, is_bf16), is_bf16)
    m = orc.rope_fraction_mask(ref, R, dA, is_bf16)
    eq, one = orc.gemm_rounded_fractions(bits(got[m], is_bf16), ref[m], is_bf16)
    _, dA_max = orc.rope_plain_angle_np(base, D, np.arange(D // 2), 131071)
    print(f"C oracle rope_append D {D} base {base:g}: worst err/budget {worst:.3f}, rounded / within one step {(eq, one)} "
          f"over {m.mean():.2f} of the outputs; angle bound at position 131071 up to {dA_max.max():.3g} rad")
    assert n == 0 and eq >= orc.ROPE_MIN_ROUNDED and one >= orc.ROPE_MIN_WITHIN_ONE


EX_CASES = [
    ("base scale 4", dict(BASE, scale=4.0), {}),
    ("llama3", dict(BASE, style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192), {}),
    ("yarn", dict(BASE, style=5, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13), {}),
    ("dynamic ntk", dict(BASE, style=3, scale=2.0, max_pos=512), {}),
    ("qwen ntk", dict(BASE, style=4, max_pos=1024), dict(pos=[1023, 1024, 2046, 2047, 2048, 4094, 4095, 4096, 131071])),
    ("cache boundary", dict(BASE, scale=1.0), dict(cache=64, pos=[0, 5, 63, 64, 65, 131071])),
    ("partial dim + bias + logn", dict(BASE, dim=64, max_pos=16), dict(bias=True, logn=True, pos=[0, 15, 16, 17, 2049, 131071])),
]


def ex_case(is_bf16, cfg, opt, seed=1):
    rng = np.random.default_rng(seed)
    pos = np.asarray(opt.get("pos", POSITIONS), np.int32)
    B, Hq, Hkv, D, T = len(pos), 4, 2, 128, 16
    qkv = orc.round_t(rng.standard_normal((B, (Hq + 2 * Hkv) * D)), is_bf16)
    bias = orc.round_t(rng.standard_normal((Hq + 2 * Hkv) * D) * 0.1, is_bf16) if opt.get("bias") else None
    cache = orc.rope_cache_base(cfg["dim"], cfg["base"], 2.0, opt["cache"] // 2) if opt.get("cache") else None
    return dict(qkv=qkv, bias=bias, cache=cache, pos=pos, Hq=Hq, Hkv=Hkv, D=D, T=T, cfg=cfg, logn=bool(opt.get("logn")))


def c_rope_ex(e, is_bf16):
    B, T = len(e["pos"]), e["T"]
    M = int(e["pos"].max()) // T + 1
    block_ids = np.zeros((B, M), np.int32)
    block_ids[np.arange(B), e["pos"] // T] = 1 + np.arange(B)
    pool = np.zeros((1 + B, 2, e["Hkv"], T, e["D"]), np.uint16)
    q, pool = orc.rope_append_ex(bits(e["qkv"], is_bf16), pool, orc.convert_block_table(block_ids), e["pos"], e["Hq"], e["Hkv"], e["D"],
                                 T, e["cfg"], bias_bits=None if e["bias"] is None else bits(e["bias"], is_bf16),
                                 cos_sin_cache=e["cache"], use_logn=e["logn"], is_bf16=is_bf16)
    kv = pool[1 + np.arange(B), :, :, e["pos"] % T]
    out = np.concatenate([q.reshape(B, e["Hq"], e["D"]), kv[:, 0], kv[:, 1]], 1)
    return orc.from_bits(out, is_bf16).astype(np.float64)


def ex_ref(e, is_bf16):
    return orc.rope_np(e["qkv"], e["Hq"], e["Hkv"], e["D"], e["pos"], cfg=e["cfg"], bias=e["bias"], cos_sin_cache=e["cache"],
                       use_logn=e["logn"], is_bf16=is_bf16)


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", EX_CASES, ids=[c[0] for c in EX_CASES])
def test_c_oracle_rope_append_ex_within_budget(is_bf16, case):
    name, cfg, opt = case
    e = ex_case(is_bf16, cfg, opt)
    got = c_rope_ex(e, is_bf16)
    ref, R, dA = ex_ref(e, is_bf16)
    n, worst = violations(got, ref, orc.rope_error_budget(ref, R, dA, is_bf16), is_bf16)
    print(f"C oracle rope_append_ex '{name}': worst err/budget {worst:.3f}")
    assert n == 0


def rotate(x, a, D, dim=None):
    """NeoX rotation of [B, H, D] by angles a [B, dim / 2]."""
    dim = dim or D
    h = dim // 2
    out = x.copy()
    c, s = np.cos(a)[:, None], np.sin(a)[:, None]
    out[..., :h] = x[..., :h] * c - x[..., h:dim] * s
    out[..., h:dim] = x[..., h:dim] * c + x[..., :h] * s
    return out


def rope_mutant(name, is_bf16):
    """(mutant output [B, H, D] rounded to T, ref, R, dA, fraction mask or None)"""
    if name in ("position + 1", "position - 1", "position through fp16", "interleaved pairing"):
        pos = np.array([1, 2, 15, 16, 2049, 2051, 4097, 8191, 32767, 65533], np.int32)
        qkv, c = plain_case(is_bf16, positions=pos)
        ref, R, dA = orc.rope_np(qkv, c["Hq"], c["Hkv"], c["D"], pos, base=c["base"], is_bf16=is_bf16)
        x = qkv.reshape(len(pos), -1, c["D"])
        H = c["Hq"] + c["Hkv"]
        i = np.arange(c["D"] // 2)
        if name == "interleaved pairing":
            perm = np.concatenate([np.arange(0, c["D"], 2), np.arange(1, c["D"], 2)])
            xr = x.copy()
            xr[:, :H] = rotate(x[:, :H][..., perm], orc.rope_plain_angle_np(c["base"], c["D"], i, pos[:, None])[0], c["D"])[..., np.argsort(perm)]
        else:
            xr = x.copy()
            with np.errstate(over="ignore", invalid="ignore"):       # fp16 has no 65533: it becomes inf, the output NaN
                p = {"position + 1": pos + 1.0, "position - 1": pos - 1.0,
                     "position through fp16": pos.astype(np.float16).astype(np.float64)}[name]
                xr[:, :H] = rotate(x[:, :H], orc.rope_plain_angle_np(c["base"], c["D"], i, p[:, None])[0], c["D"])
        return orc.round_t(xr, is_bf16), ref, R, dA, None
    if name == "bias not rounded to T":
        e = ex_case(is_bf16, BASE, dict(bias=True, pos=np.arange(0, 40, 3)))
        ref, R, dA = ex_ref(e, is_bf16)
        raw = e["qkv"] + e["bias"]                                             # x + b kept in full precision
        mut = orc.rope_np(raw, e["Hq"], e["Hkv"], e["D"], e["pos"], cfg=e["cfg"])[0]
        return orc.round_t(mut, is_bf16), ref, R, dA, orc.rope_fraction_mask(ref, R, dA, is_bf16)
    if name == "logn at pos >= max_pos":
        e = ex_case(is_bf16, dict(BASE, max_pos=16), dict(logn=True, pos=[3, 15, 16, 16, 17, 40]))
        ref, R, dA = ex_ref(e, is_bf16)
        mut = ref.copy()
        at = e["pos"] == 16
        mut[at, :e["Hq"]] *= np.log(17.0) / np.log(16.0)
        return orc.round_t(mut, is_bf16), ref, R, dA, None
    if name == "cache used at pos == cache_positions":
        e = ex_case(is_bf16, BASE, dict(cache=64, pos=[0, 63, 64, 64, 64]))
        ref, R, dA = ex_ref(e, is_bf16)
        e["cache"] = orc.rope_cache_base(BASE["dim"], BASE["base"], 2.0, 33)          # 66 rows: row 64 now exists
        return orc.round_t(ex_ref(e, is_bf16)[0], is_bf16), ref, R, dA, None
    if name == "Qwen-NTK step one position early":
        cfg = dict(BASE, style=4, max_pos=1024)
        e = ex_case(is_bf16, cfg, dict(pos=[1022, 1023, 2046, 2047, 4094, 4095]))
        ref, R, dA = ex_ref(e, is_bf16)
        i = np.arange(cfg["dim"] // 2)
        a = orc.rope_angle_np(cfg, 2 * i[None, :], e["pos"][:, None], seq_len=e["pos"][:, None] + 2.0)[0]
        x = e["qkv"].reshape(len(e["pos"]), -1, e["D"])
        mut = x.copy()
        H = e["Hq"] + e["Hkv"]
        mut[:, :H] = rotate(x[:, :H], a, e["D"], cfg["dim"])
        return orc.round_t(mut, is_bf16), ref, R, dA, None
    raise ValueError(name)


ROPE_MUTANTS = ["position + 1", "position - 1", "position through fp16", "interleaved pairing", "bias not rounded to T",
                "logn at pos >= max_pos", "cache used at pos == cache_positions", "Qwen-NTK step one position early"]


@pytest.mark.parametrize("is_bf16", [False, True], ids=["f16", "bf16"])
@pytest.mark.parametrize("name", ROPE_MUTANTS)
def test_rope_mutant_is_rejected(is_bf16, name):
    mut, ref, R, dA, mask = rope_mutant(name, is_bf16)
    n, worst = violations(mut, ref, orc.rope_error_budget(ref, R, dA, is_bf16), is_bf16)
    msg = f"rope mutant '{name}': {n} outputs outside the budget (worst {worst:.3g})"
    if mask is not None:
        eq, one = orc.gemm_rounded_fractions(bits(mut[mask], is_bf16), ref[mask], is_bf16)
        msg += f", rounded / within one step {(eq, one)} over {mask.mean():.2f} of the outputs"
        caught = n > 0 or eq < orc.ROPE_MIN_ROUNDED or one < orc.ROPE_MIN_WITHIN_ONE
    else:
        caught = n > 0
    print(msg)
    assert caught
