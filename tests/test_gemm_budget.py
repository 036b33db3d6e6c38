"""The weight-only GEMM's float64 reference, error budget and rounded-fraction check (oracle.round_t, dequant_exact, gemm_np,
gemm_error_budget, gemm_rounded_fractions), without a GPU: the single rounding to fp16 / bf16 at ties, subnormals and
overflow, hand-computed dequantised weights, and, at the Llama-3-8B w2 shape, a simulated fp32 kernel that passes both
checks next to four subtly wrong kernels that each fail one of them."""
import numpy as np
import pytest

from oracle import oracle as orc


def bf16_value(bits):
    return orc.bf16_bits_to_f32(np.asarray(bits, np.uint16)).astype(np.float64)


# ---------------------------------------------------------------------------------------------- rounding to T
def test_bf16_rounding_of_every_bf16_value_and_midpoint():
    """Every finite bf16 value rounds to itself; the midpoint between two neighbours goes to the even one; a hair above or
    below it goes to the nearer one (also where a float32 cast would first round the hair away)."""
    b = np.arange(0, 0x7F80, dtype=np.uint32).astype(np.uint16)          # every finite non-negative bf16, subnormals included
    v = bf16_value(b)
    for sign in (1.0, -1.0):
        assert np.array_equal(orc.f64_to_bits(sign * v, True), b | (np.uint16(0x8000) if sign < 0 else np.uint16(0)))
    lo, hi = v[:-1], v[1:]
    mid = (lo + hi) / 2                                                    # exact in float64
    even = np.where(b[:-1] % 2 == 0, b[:-1], b[1:])
    assert np.array_equal(orc.f64_to_bits(mid, True), even)
    up, down = np.nextafter(mid, np.inf), np.nextafter(mid, -np.inf)
    assert np.array_equal(orc.f64_to_bits(up, True), b[1:])
    assert np.array_equal(orc.f64_to_bits(down, True), b[:-1])
    # 1 + 2^-8 + 2^-30: above the bf16 midpoint of 1 and 1 + 2^-7, but float32 rounds it to the midpoint, which ties to 1
    x = 1.0 + 2.0 ** -8 + 2.0 ** -30
    assert orc.f64_to_bits(x, True) == 0x3F81
    assert orc.f32_to_bf16_bits(np.float32(x)) == 0x3F80


def test_bf16_rounding_edges():
    big = float(bf16_value(0x7F7F))                                        # largest finite bf16
    half = 2.0 ** (127 - 8)                                                # half its ulp
    cases = [(0.0, 0x0000), (-0.0, 0x8000), (2.0 ** -133, 0x0001), (2.0 ** -134, 0x0000), (2.0 ** -134 * 1.5, 0x0001),
             (3 * 2.0 ** -134, 0x0002), (2.0 ** -126, 0x0080), (2.0 ** -126 - 2.0 ** -134, 0x0080), (big, 0x7F7F),
             (big + half - 2.0 ** 100, 0x7F7F), (big + half, 0x7F80), (-(big + half), 0xFF80), (np.inf, 0x7F80), (-np.inf, 0xFF80)]
    for x, want in cases:
        assert int(orc.f64_to_bits(np.float64(x), True)) == want, (x, hex(int(orc.f64_to_bits(np.float64(x), True))), hex(want))
    assert np.isnan(orc.round_t(np.nan, True))


def test_fp16_rounding_matches_numpys_single_rounding():
    rng = np.random.default_rng(0)
    b = np.arange(0, 0x7C00, dtype=np.uint16)
    v = b.view(np.float16).astype(np.float64)
    mid = (v[:-1] + v[1:]) / 2
    x = np.concatenate([v, -v, mid, -mid, np.nextafter(mid, np.inf), np.nextafter(mid, -np.inf),
                        rng.standard_normal(100000) * 10.0 ** rng.uniform(-9, 5, 100000), [65504.0, 65519.99, 65520.0, 1e6]])
    with np.errstate(over="ignore"):                                       # 1e6 overflows to inf, as it should
        assert np.array_equal(orc.f64_to_bits(x, False), x.astype(np.float16).view(np.uint16))


# ---------------------------------------------------------------------------------------------- dequant_exact
def test_dequant_exact_by_hand():
    # int4: low nibble = even column. q_s = -8, 7 | 1, -1; group 2 (k 0, 1 share row 0 of s / zs)
    w = np.array([[0x78], [0xF1]], np.uint8)                              # k0: cols (8 -> -8, 7); k1: cols (1, -1)
    s = np.array([[0.5, 2.0 ** -13]], np.float64)
    zs = np.array([[3.0, -(2.0 ** -20)]], np.float64)
    got = orc.dequant_exact("int4", w, s, zs, group=2)
    # col 1: 7 * 2^-13 - 2^-20 = (896 - 1) * 2^-20 = 895 * 2^-20: 10 significant bits, exact in fp16
    assert got.tolist() == [[-8 * 0.5 + 3.0, 895 * 2.0 ** -20], [0.5 + 3.0, -(2.0 ** -13) - 2.0 ** -20]]
    # a value that needs rounding, once: 1 * 1.0009765625 + 2^-11: the exact sum sits half an fp16 ulp above 1 + 2^-10
    w1 = np.array([[0x01]], np.uint8)                                      # col 0: q 1, col 1: q 0
    s1 = np.array([[1.0 + 2.0 ** -10, 1.0]])
    z1 = np.array([[2.0 ** -11, 0.0]])
    assert orc.dequant_exact("int4", w1, s1, z1, group=1)[0, 0] == 1.0 + 2.0 ** -9    # tie -> even
    # bf16: 1 + 2^-8 is the midpoint of 1 and 1 + 2^-7 -> 1 (even); with 2^-40 more it rounds up
    w8 = np.array([[1, 1]], np.int8)
    s8 = np.array([[1.0, 1.0]])
    z8 = np.array([[2.0 ** -8, 2.0 ** -8 + 2.0 ** -40]])
    assert orc.dequant_exact("int8g", w8, s8, z8, group=1, is_bf16=True).tolist() == [[1.0, 1.0 + 2.0 ** -7]]
    # fp16 subnormal through the zero*scale rounding: q s + zs = 2^-30 * 3 -> rounds to 0 (below half of 2^-24)
    assert orc.dequant_exact("int8g", np.array([[1]], np.int8), np.array([[2.0 ** -10]]),
                             np.array([[-(2.0 ** -10) + 3 * 2.0 ** -30]]), group=1)[0, 0] == 0.0
    assert orc.dequant_exact("int8g", np.array([[1]], np.int8), np.array([[2.0 ** -10]]),
                             np.array([[-(2.0 ** -10) + 3 * 2.0 ** -25]]), group=1)[0, 0] == 2.0 ** -23
    # int8 per-column: q itself; f16: the values, or their bits
    assert orc.dequant_exact("int8", np.array([[-128, 127]], np.int8)).tolist() == [[-128.0, 127.0]]
    wf = np.array([[0.1, -3.0]], np.float16)
    assert np.array_equal(orc.dequant_exact("f16", wf.view(np.uint16)), wf.astype(np.float64))


def test_dequant_exact_rounds_once_where_dequant_np_rounds_twice():
    """dequant_np takes the int4 value through float32 before T; dequant_exact rounds q_s * s + zs once. For bf16 a
    float32 step can land on a bf16 midpoint and then tie the wrong way."""
    w = np.array([[1, 1]], np.int8)
    s = np.array([[1.0, 1.0]], np.float32)
    z = np.array([[2.0 ** -8 + 2.0 ** -30, 2.0 ** -8]], np.float64)      # not float32 values: only dequant_exact sees the tail
    assert orc.dequant_exact("int8g", w, s, z, group=1, is_bf16=True)[0].tolist() == [1.0 + 2.0 ** -7, 1.0]
    assert orc.dequant_np("int8g", w, s, z, group=1, is_bf16=True)[0].tolist() == [1.0, 1.0]


def test_gemm_np_terms():
    x = np.array([[1.0, -2.0]])
    w = np.array([[3.0, 0.5], [1.0, -4.0]])
    ref, A = orc.gemm_np(x, w, cscale=np.array([2.0, -1.0]), bias=np.array([0.25, 1.0]))
    assert ref.tolist() == [[(3 - 2) * 2 + 0.25, (0.5 + 8) * -1 + 1.0]]
    assert A.tolist() == [[(3 + 2) * 2 + 0.25, (0.5 + 8) * 1 + 1.0]]


def test_rounded_fractions_count_steps():
    ref = np.array([1.0, 1.0 + 2.0 ** -10, -1.0, 0.0, 3.0])
    got = np.array([1.0, 1.0, -1.0 - 2.0 ** -10, -0.0, 3.0 + 2 * 2.0 ** -9]).astype(np.float16)
    eq, one = orc.gemm_rounded_fractions(got, ref, False)
    assert (eq, one) == (2 / 5, 4 / 5)
    # across a binade: 1 - 2^-11 and 1 are neighbours
    assert orc.gemm_rounded_fractions(np.array([1.0 - 2.0 ** -11], np.float16), np.array([1.0]), False) == (0.0, 1.0)


# ---------------------------------------------------------------------------------------------- the worst-case adder
def truncating_step(acc, products):
    """One k16 step of a 24-bit adder without guard bits: the accumulator and the 16 products aligned to the largest
    exponent E, each truncated toward zero to a multiple of 2^(E-23), summed, and the sum truncated to 24 bits."""
    addends = np.concatenate([[acc], products])
    E = np.floor(np.log2(np.abs(addends).max()))
    q = 2.0 ** (E - 23)
    s = float(np.sum(np.trunc(addends / q) * q))                          # exact: multiples of q, far below 2^53 q
    if s == 0.0:
        return 0.0
    qs = 2.0 ** (np.floor(np.log2(abs(s))) - 23)
    return float(np.trunc(s / qs) * qs)


def test_budget_covers_a_truncating_adder():
    """The bound's model, played adversarially: a large accumulator and 16 products each just under the alignment step,
    so every product loses almost all of itself. Every step loses nearly 16 * 2^-23 of the sum; the chain stays within
    gemm_fp32_error (which a bound of 2 * 2^-23 per step would not)."""
    kb = 4                                                                # 32 k16 steps, one split
    acc, exact, A = 1.0, 1.0, 1.0
    small = (1 - 2.0 ** -11) * 2.0 ** -23
    for _ in range(8 * kb):
        p = np.full(16, small)
        acc = truncating_step(acc, p)
        exact += p.sum()
        A += p.sum()
    err = exact - acc
    assert err > 8 * kb * 15 * 2.0 ** -24                                 # the model's worst case is real: far above 2 * 2^-23 per step
    assert err <= orc.gemm_fp32_error(np.array(A), 128 * kb, 1)


# ---------------------------------------------------------------------------------------------- mutants at the w2 shape
B, K, N, NSPLIT = 32, 14336, 4096, 8          # Llama-3-8B w2 at batch 32; 8 splits of 14 k-blocks (the library's plan there)


def simulate(x, w, nsplit, is_bf16, round_partials=False, drop_step=None):
    """A kernel as the contract describes it, in numpy: each split accumulates its k16 steps in fp32 (16 exact products and
    the accumulator summed, rounded to nearest once per step), the partials are summed in split order in fp32, and the sum is
    rounded once to T. round_partials: each partial is first rounded to T (the mutant). drop_step = (k16 step, tile): that
    step's products are left out of that 128-feature tile."""
    kb = K // 128
    kbp = -(-kb // nsplit)
    total = np.zeros((x.shape[0], w.shape[1]), np.float32)
    for s in range(nsplit):
        acc = np.zeros_like(total)
        for j in range(s * kbp * 8, min(kb, (s + 1) * kbp) * 8):
            step = x[:, 16 * j:16 * j + 16] @ w[16 * j:16 * j + 16]
            if drop_step is not None and drop_step[0] == j:
                t = drop_step[1]
                step[:, 128 * t:128 * t + 128] = 0.0
            acc = (acc.astype(np.float64) + step).astype(np.float32)
        if round_partials:
            acc = orc.round_t(acc, is_bf16).astype(np.float32)
        total = total + acc
    return orc.round_t(total.astype(np.float64), is_bf16)


def checks(y, ref, A, is_bf16):
    """(within the budget everywhere, rounded fractions above the thresholds, worst err/budget, fractions)"""
    ratio = np.abs(y - ref) / orc.gemm_error_budget(ref, A, K, NSPLIT, is_bf16)
    eq, one = orc.gemm_rounded_fractions(y, ref, is_bf16)
    return bool(ratio.max() <= 1.0), eq >= orc.GEMM_MIN_ROUNDED and one >= orc.GEMM_MIN_WITHIN_ONE, float(ratio.max()), (eq, one)


@pytest.fixture(scope="module", params=[False, True], ids=["f16", "bf16"])
def w2(request):
    """The suite's realistic INT4 w2 weight (tests/gpu_probe.make_w4's distribution) and N(0, 1) activations in T."""
    is_bf16 = request.param
    rng = np.random.default_rng(2)
    qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
    s = orc.round_t(np.abs(rng.standard_normal((K // 128, N))) * 0.01 + 1e-3, is_bf16)
    zs = orc.round_t((8 - rng.integers(0, 16, (K // 128, N))) * s, is_bf16)
    x = orc.round_t(rng.standard_normal((B, K)), is_bf16)
    w = orc.dequant_exact("int4", qp, s, zs, is_bf16=is_bf16)
    ref, A = orc.gemm_np(x, w)
    return dict(is_bf16=is_bf16, qp=qp, s=s, zs=zs, x=x, w=w, ref=ref, A=A, rng=rng)


def test_fp32_kernel_passes(w2):
    y = simulate(w2["x"], w2["w"], NSPLIT, w2["is_bf16"])
    ok_budget, ok_frac, worst, fr = checks(y, w2["ref"], w2["A"], w2["is_bf16"])
    print(f"simulated fp32 kernel: worst err/budget {worst:.3f}, rounded / within one step {fr}")
    assert ok_budget and ok_frac, (worst, fr)
    y1 = simulate(w2["x"], w2["w"], 1, w2["is_bf16"])                     # unsplit: one chain of 896 steps
    assert checks(y1, w2["ref"], w2["A"], w2["is_bf16"])[:2] == (True, True)


def _mutant(w2, name):
    x, is_bf16 = w2["x"], w2["is_bf16"]
    if name == "split partials rounded to T":
        return simulate(x, w2["w"], NSPLIT, is_bf16, round_partials=True)
    if name == "one zero point off by one step":
        zs = w2["zs"].copy()
        g, n = 57, 1234
        zs[g, n] = orc.round_t(zs[g, n] + w2["s"][g, n], is_bf16)
        return simulate(x, orc.dequant_exact("int4", w2["qp"], w2["s"], zs, is_bf16=is_bf16), NSPLIT, is_bf16)
    if name == "one k16 step dropped in one tile":
        return simulate(x, w2["w"], NSPLIT, is_bf16, drop_step=(333, 17))
    if name == "W' rounded twice":
        q = orc.unpack_int4_signed(w2["qp"]).astype(np.float64)
        s, z = np.repeat(w2["s"], 128, axis=0), np.repeat(w2["zs"], 128, axis=0)
        return simulate(x, orc.round_t(orc.round_t(q * s, is_bf16) + z, is_bf16), NSPLIT, is_bf16)
    raise ValueError(name)


@pytest.mark.parametrize("name", ["split partials rounded to T", "one zero point off by one step", "one k16 step dropped in one tile",
                                  "W' rounded twice"])
def test_mutant_is_rejected(w2, name):
    ok_budget, ok_frac, worst, fr = checks(_mutant(w2, name), w2["ref"], w2["A"], w2["is_bf16"])
    print(f"{name}: worst err/budget {worst:.3f}, rounded / within one step {fr}")
    assert not (ok_budget and ok_frac), (worst, fr)
