"""GPU tests (H100) of b200_constrain_logits against the bit-exact numpy contract (tests/constrain_oracle.py) per logits dtype,
across vocabularies, row counts, mask kinds, strides and biases; on an unaligned row base; behind the lm_head GEMM under PDL in
a CUDA graph with new masks copied in between replays; inside a decode program; the endings on a fully masked row; and
b200_sample's min-p kept set, exactly, against the kernel's own probabilities."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from tests.constrain_oracle import BITS, NEG_INF, constrain, min_p_kept, round_to  # noqa: E402
from tests.test_gpu_sampler_edges import VOCABS, _batch_inputs, _filtered_row  # noqa: E402

dev = torch.device("cuda")
TORCH_DT = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}
INT_DT = {"fp16": torch.int16, "bf16": torch.int16, "fp32": torch.int32}
NAN_BITS = {"fp16": 0x7E01, "bf16": 0x7FC1, "fp32": 0x7FC00123}       # quiet NaNs with a payload the kernel must keep
KINDS = ["ones", "zeros", "first", "last", "word_end", "word_start", "rand1", "rand50", "rand99"]


def to_dev(bits, dtype, out=None):
    t = torch.from_numpy(np.ascontiguousarray(bits).view(np.int32 if dtype == "fp32" else np.int16)).to(dev).view(TORCH_DT[dtype])
    if out is None:
        return t
    out.copy_(t)
    return out


def from_dev(t, dtype):
    return t.view(INT_DT[dtype]).cpu().numpy().view(BITS[dtype])


def random_logits(rows, V, dtype, rng):
    x = (rng.standard_normal((rows, V)) * 3).astype(np.float32)
    bits = round_to(x, dtype)
    pick = rng.random((rows, V))
    bits[pick < 1e-3] = NAN_BITS[dtype]
    bits[(pick >= 1e-3) & (pick < 2e-3)] = round_to(np.float32(np.inf), dtype)
    bits[(pick >= 2e-3) & (pick < 3e-3)] = NEG_INF[dtype]
    return bits


def make_mask(kinds, V, stride, rng):
    """int32 [rows, stride]: each row's allowed set by kind, garbage in the bits past V and in the words past ceil(V / 32)."""
    words = (V + 31) // 32
    m = rng.integers(0, 1 << 32, (len(kinds), stride), dtype=np.uint64).astype(np.uint32)
    weights = np.uint64(1) << np.arange(32, dtype=np.uint64)
    for r, k in enumerate(kinds):
        a = np.zeros(words * 32, bool)
        if k == "ones":
            a[:V] = True
        elif k == "first":
            a[0] = True
        elif k == "last":
            a[V - 1] = True
        elif k == "word_end":                    # either side of a word boundary
            a[min(31, V - 1)] = True
        elif k == "word_start":
            a[min(32, V - 1)] = True
        elif k.startswith("rand"):
            a[:V] = rng.random(V) < int(k[4:]) / 100
        w = (a.reshape(words, 32) * weights).sum(axis=1).astype(np.uint32)
        if V % 32:                               # keep the garbage past V in the last word
            w[-1] |= m[r, words - 1] & ~np.uint32((1 << (V % 32)) - 1)
        m[r, :words] = w
    return m.view(np.int32)


def make_bias(rows, V, rng, per_row=300):
    """Odd rows: per_row distinct ids (masked and allowed tokens alike, and 5 outside [0, V)) with values that include -inf
    and fp16-overflowing ones; even rows: none."""
    offsets, ids, values = [0], [], []
    for r in range(rows):
        if r % 2:
            inside = rng.choice(V, min(per_row - 5, V), replace=False)
            t = np.concatenate([inside, [-1, -7, V, V + 5, 2 ** 31 - 1]])
            v = (rng.standard_normal(t.size) * 5).astype(np.float32)
            v[:3] = [-np.inf, 7e4, -7e4]
            ids += t.tolist()
            values += v.tolist()
        offsets.append(len(ids))
    return np.array(offsets, np.int32), np.array(ids, np.int32), np.array(values, np.float32)


def is_nan(bits, dtype):
    if dtype == "fp32":
        return np.isnan(bits.view(np.float32))
    return (bits & 0x7FFF) > (0x7C00 if dtype == "fp16" else 0x7F80)


def assert_bits(got, exp, biased, dtype, what):
    """Every logit's bits equal the oracle's; a biased logit whose result is NaN only has to be NaN."""
    bad = (got != exp) & ~(biased & is_nan(exp, dtype) & is_nan(got, dtype))
    if bad.any():
        r, t = np.argwhere(bad)[0]
        pytest.fail(f"{what}: {bad.sum()} logits differ, first at row {r} token {t}: {got[r, t]:#x} vs {exp[r, t]:#x}")


def _bias_dev(bias):
    return tuple(torch.from_numpy(a).to(dev) for a in bias)


@pytest.mark.parametrize("rows", [1, 7, 32, 128])
@pytest.mark.parametrize("V", [1000, 32000, 50257, 128256, 151936])
@pytest.mark.parametrize("dtype", ["fp16", "bf16", "fp32"])
def test_constrain_matches_the_contract(dtype, V, rows):
    rng = np.random.default_rng(V + rows)
    words = (V + 31) // 32
    stride = words + (3 if rows in (7, 128) else 0)
    kinds = [KINDS[(i + rows) % len(KINDS)] for i in range(rows)]
    bits = random_logits(rows, V, dtype, rng)
    mask = make_mask(kinds, V, stride, rng)
    bias = make_bias(rows, V, rng)
    for with_mask in (True, False):
        x = to_dev(bits, dtype)
        ops.constrain_logits(x, torch.from_numpy(mask).to(dev) if with_mask else None, _bias_dev(bias))
        exp, biased = constrain(bits, dtype, mask if with_mask else None, *bias)
        assert_bits(from_dev(x, dtype), exp, biased, dtype, f"{dtype} V={V} rows={rows} mask={with_mask}")
    if rows == 128:
        assert set(kinds) == set(KINDS)


@pytest.mark.parametrize("dtype", ["fp16", "fp32"])
def test_unaligned_rows_take_the_scalar_stores(dtype):
    rows, V = 9, 4096
    rng = np.random.default_rng(1)
    bits = random_logits(rows, V, dtype, rng)
    mask = make_mask([KINDS[i] for i in range(rows)], V, V // 32, rng)
    base = torch.empty(rows * V + 8, dtype=TORCH_DT[dtype], device=dev)
    x = base[1:1 + rows * V].view(rows, V)                                  # one element past a 16-byte boundary
    to_dev(bits, dtype, out=x)
    bias = make_bias(rows, V, rng)
    ops.constrain_logits(x, torch.from_numpy(mask).to(dev), _bias_dev(bias))
    exp, biased = constrain(bits, dtype, mask, *bias)
    assert_bits(from_dev(x, dtype), exp, biased, dtype, f"{dtype} unaligned")


def test_fully_masked_rows_in_the_endings():
    """A row whose mask allows nothing is all -inf: b200_argmax returns 0, b200_sample -1 with probability 0."""
    V = 1000
    x = torch.randn(3, V, device=dev)
    m = np.zeros((3, 32), np.int32)
    m[1, 517 >> 5] = 1 << (517 & 31)
    m[2] = -1
    ops.constrain_logits(x, torch.from_numpy(m).to(dev))
    assert torch.isneginf(x[0]).all() and torch.isneginf(x[1]).sum() == V - 1
    am = ops.argmax(x)
    assert am.tolist()[:2] == [0, 517]
    tok, tprob, _ = ops.sample(x.clone(), torch.zeros(3, dtype=torch.int32, device=dev), torch.ones(3, device=dev),
                               torch.full((3,), 0.5, device=dev))
    assert tok.tolist()[:2] == [-1, 517] and float(tprob[0]) == 0.0 and float(tprob[1]) == 1.0


def test_graph_replay_with_pdl_behind_the_lm_head_and_new_masks_between_replays():
    B, K, V = 32, 4096, 128256
    gen = torch.Generator(device=dev).manual_seed(3)
    xin = torch.randn(B, K, generator=gen, device=dev).half()
    w = ops.pack_f16((torch.randn(K, V, generator=gen, device=dev) * 0.05).half())
    ws = ops.gemm_workspace(B, [(K, V)], dev)
    y = torch.empty(B, V, dtype=torch.float16, device=dev)
    ops.wo_gemm(xin, w, ws, out=y)
    torch.cuda.synchronize()
    raw = from_dev(y, "fp16")
    words, cap = (V + 31) // 32, 300 * B
    mask = torch.empty(B, words, dtype=torch.int32, device=dev)
    bias = (torch.zeros(B + 1, dtype=torch.int32, device=dev), torch.zeros(cap, dtype=torch.int32, device=dev),
            torch.zeros(cap, device=dev))
    rng = np.random.default_rng(5)

    def fill(i):
        m = make_mask([KINDS[(r + i) % len(KINDS)] for r in range(B)], V, words, rng)
        b = make_bias(B, V, rng)
        mask.copy_(torch.from_numpy(m))
        bias[0].copy_(torch.from_numpy(b[0]))
        bias[1][:b[1].size].copy_(torch.from_numpy(b[1]))
        bias[2][:b[2].size].copy_(torch.from_numpy(b[2]))
        return m, b

    def chain():
        ops.wo_gemm(xin, w, ws, out=y, pdl=True)
        ops.constrain_logits(y, mask, bias)

    try:
        ops.set_pdl(True)
        fill(0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            chain()
        for i in range(3):
            m, b = fill(i + 1)
            y.fill_(float("nan"))
            graph.replay()
            torch.cuda.synchronize()
            exp, biased = constrain(raw, "fp16", m, b[0], b[1], b[2])
            assert_bits(from_dev(y, "fp16"), exp, biased, "fp16", f"fp16 graph replay {i}")
    finally:
        ops.set_pdl(False)


def test_inside_a_decode_program():
    rows, V = 16, 32000
    rng = np.random.default_rng(9)
    bits = random_logits(rows, V, "bf16", rng)
    x = to_dev(bits, "bf16")
    mask = torch.empty(rows, V // 32, dtype=torch.int32, device=dev)
    bias = _bias_dev(make_bias(rows, V, rng))
    prog = ops.Program()
    with prog.record():
        ops.constrain_logits(x, mask, bias)
    assert prog.num_launches == 1
    for i in range(2):                                                      # a new mask each launch: the pointers are frozen
        m = make_mask([KINDS[(r + i) % len(KINDS)] for r in range(rows)], V, V // 32, rng)
        mask.copy_(torch.from_numpy(m))
        to_dev(bits, "bf16", out=x)
        prog.launch()
        torch.cuda.synchronize()
        exp, biased = constrain(bits, "bf16", m, *(t.cpu().numpy() for t in bias))
        assert_bits(from_dev(x, "bf16"), exp, biased, "bf16", f"bf16 program launch {i}")


# ---------------------------------------------------------------------------------------------------- min-p in b200_sample
def _t(a, dt):
    return torch.tensor(np.asarray(a), dtype=dt, device=dev)


def _near(m, n=4):
    """m and the n floats on either side of it."""
    out = [m]
    lo = hi = m
    for _ in range(n):
        lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(2))
        out += [lo, hi]
    return out


@pytest.mark.parametrize("V", [1000, 32000, 128256])
def test_min_p_keeps_exactly_the_tokens_at_or_above_the_bound(V):
    rng = np.random.default_rng(V)
    #        top_k, top_p, min_p (None: set below to land exactly on a probability)
    rows = [(0, 1.0, 0.05), (0, 1.0, 0.5), (0, 1.0, 1.0), (50, 1.0, 0.1), (0, 0.9, 0.2), (20, 0.8, 0.3), (1, 1.0, 0.5),
            (0, 1.0, None), (40, 0.95, None), (0, 1.0, 1e-3)]
    n = len(rows)
    lg = (rng.standard_normal((n, V)) * 2).astype(np.float32)
    lg[:, rng.choice(V, 6, replace=False)] = lg.max() + 0.5                  # tied maxima
    lg[:, rng.choice(V, 40, replace=False)] = lg.max() - 1.0                 # a tie group below them
    top_k, top_p = _t([r[0] for r in rows], torch.int32), _t([r[1] for r in rows], torch.float32)
    u = _t(rng.random(n), torch.float32)
    xa = torch.from_numpy(lg).to(dev)
    tok_a, _, probs_a = ops.sample(xa, top_k, top_p, u, want_probs=True)
    pa = xa.cpu().numpy()
    base = probs_a.cpu().numpy() > 0
    mp = np.array([r[2] if r[2] is not None else 0.0 for r in rows], np.float32)
    pmax = pa.max(axis=1)
    for i, r in enumerate(rows):
        if r[2] is None:                       # a bound equal to a kept probability below the max: that token stays
            cand = np.unique(pa[i][base[i] & (pa[i] < pmax[i])])
            for q in cand[::-1]:
                hits = [m for m in _near(np.float32(q / pmax[i])) if np.float32(m * pmax[i]) == q]
                if hits:
                    mp[i] = hits[0]
                    break
            assert mp[i] > 0, f"row {i}: no probability is an exact product"
    xb = torch.from_numpy(lg).to(dev)
    tok, tprob, probs = ops.sample(xb, top_k, top_p, u, want_probs=True, min_p=_t(mp, torch.float32))
    assert torch.equal(xa.view(torch.int32), xb.view(torch.int32)), "min-p changed the probabilities"
    kept = probs.cpu().numpy() > 0
    exp = min_p_kept(pa, base, mp)
    for i in range(n):
        assert np.array_equal(kept[i], exp[i]), (f"row {i} {rows[i]} min_p {mp[i]!r}: kept {kept[i].sum()} vs "
                                                 f"{exp[i].sum()}, first difference at {np.flatnonzero(kept[i] != exp[i])[:4]}")
        assert exp[i][int(tok[i])], f"row {i}: drawn token {int(tok[i])} is not kept"
    exact = [i for i, r in enumerate(rows) if r[2] is None]
    for i in exact:                            # the token at the bound is in the kept set
        assert kept[i][pa[i] == np.float32(mp[i] * pmax[i])].all()
    assert int(tok[6]) == int(np.flatnonzero(pa[6] == pmax[6])[0]), "top_k 1 with min-p: the lowest index among the maxima"
    assert kept[2].sum() == (pa[2] == pmax[2]).sum()                         # min_p 1 keeps the maxima only


def _run(x, args, **kw):
    x = x.clone()
    tok, tprob, probs = ops.sample(x, *args, want_probs=True, **kw)
    torch.cuda.synchronize()
    return [t.view(torch.int32) if t.dtype == torch.float32 else t for t in (x, probs, tok, tprob)]


def test_min_p_off_is_bit_identical():
    """min_p None and min_p all zeros: the same bits of token_out, token_prob_out, probs_out and the probabilities, on the
    batch and the vocabularies of tests/test_gpu_sampler_edges.py."""
    B, V = 1024, 32000
    d = _batch_inputs(B, V, 5)
    dt = dict(top_k=torch.int32, history=torch.int32, hist_len=torch.int32, process=torch.uint8)
    a = {k: _t(v, dt.get(k, torch.float32)) for k, v in d.items() if k != "lg"}
    x = torch.from_numpy(d["lg"]).to(dev)
    args = (a.pop("top_k"), a.pop("top_p"), a.pop("u"))
    off = _run(x, args, count_ws=torch.zeros(B, V, dtype=torch.int32, device=dev), **a)
    zero = _run(x, args, count_ws=torch.zeros(B, V, dtype=torch.int32, device=dev), min_p=torch.zeros(B, device=dev), **a)
    assert all(torch.equal(p, q) for p, q in zip(off, zero))
    rng = np.random.default_rng(2)
    for V in VOCABS:
        for filt in ("none", "dense", "sparse", "underflow"):
            lg, k, p, temp = _filtered_row(V, filt, rng)
            x = torch.from_numpy(lg).to(dev).expand(4, V).contiguous()
            args = (_t([k] * 4, torch.int32), _t([p] * 4, torch.float32), _t(rng.random(4), torch.float32))
            kw = {} if temp is None else dict(temperature=_t([temp] * 4, torch.float32))
            off = _run(x, args, **kw)
            zero = _run(x, args, min_p=torch.zeros(4, device=dev), **kw)
            assert all(torch.equal(p, q) for p, q in zip(off, zero)), f"V={V} {filt}"
