"""The TP peer kernels (csrc/peer_allreduce.cuh: one-shot, two-shot, fused all-reduce + residual + RMSNorm and its gather
mode, vocab-parallel argmax; b200_wo_gemm_rs, the GEMM whose epilogue pushes the reduce-scatter words) run on ONE GPU, one
rank at a time, against exact references (tests/peer_oracle.py).

The W "regions" are ordinary allocations on one device passed to the C ABI as raw pointers. A peer kernel pushes first and
then polls only its own region, so rank r runs alone once its region already holds the words its peers would have pushed.
b200_wo_gemm_rs only writes, so all W ranks run for real, one after another, into each other's regions. For every launch
the bytes that changed in every region are compared with the model's write map (which also asserts the path), no other
byte may change, and the call counter must move as documented with the finishing ticket back at 0.

Safety rule: nothing here ever waits on another kernel. Every poll loop traps after 2^24 reads, so
  1. the counter (uint32 at region + 2 * parity_stride, the ticket in the next word) is set on the host for all W regions
     and read back; the epoch every kernel of the call computes is counter + 1;
  2. before a launch that polls, BOTH parities of rank r's region, every 8-byte word, hold {poison, epoch of the call using
     that parity} (the first call's epoch where no call uses it), and only then are the modelled slots overwritten with real
     data. A poll succeeds on its first read even where the model is wrong; a wrong address reads the poison (NaN in a sum,
     +inf with an impossible token id in argmax) and fails an output check. Where kernels write into the polled area before
     the poll (the RS GEMMs before gather + norm), the host reads the parity back right before the polling launch and checks
     every word still carries the epoch, failing the test without launching if one does not;
  3. no test relies on two kernels running at the same time (W ranks on concurrent streams are out of scope);
  4. repeated calls and graph replays are refilled by the host in between, after the counter and ticket read back as
     expected."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import _lib, ops  # noqa: E402
from tests import peer_oracle as po  # noqa: E402
from tests.test_gpu_gemm_exact import make_weight, pack, plan  # noqa: E402
from tests.test_gpu_glue_exact import NORM_FRAC  # noqa: E402
from tests.test_gpu_glue_exact import report as budget_report  # noqa: E402

dev = torch.device("cuda")
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
PEER_WORD = (0x5EED5EED, 0xA5A5A5A5)      # what the regions hold outside the polled parities (a flag no call uses)
SENTINEL = 0x7E01                          # fp16 / bf16 NaN: output elements a kernel must not write


def lib():
    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def i32(a):
    """uint32 values -> an int32 device tensor with the same bits."""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.uint64).astype(np.uint32)).view(np.int32)).to(dev)


def s32(v):
    """A uint32 value as the int32 with the same bits."""
    return int(np.array(v, np.uint32).view(np.int32))


def dev_bits(bits, dtype):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint16).view(np.int16)).to(dev).view(dtype)


def bits_of(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def sentinel(shape, dtype):
    return torch.full(shape, SENTINEL, dtype=torch.int16, device=dev).view(dtype)


class Regions:
    """W peer regions on one device, the pointer array the C ABI takes, and the host side of the safety rule."""

    def __init__(self, world, max_msg):
        self.world, self.max_msg = world, max_msg
        self.lay = po.Layout(max_msg)
        nbytes = lib().b200_peer_ar_region_bytes(max_msg)
        assert nbytes == self.lay.region_bytes
        self.buf = [torch.empty(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
        self.ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in self.buf])

    def w32(self, q):
        return self.buf[q].view(torch.int32)

    def prefill(self, counter, polled, epochs, poison):
        """Every region: PEER_WORD words and call counter `counter` (ticket 0), read back. Regions of the ranks in `polled`:
        both parities {poison, epoch}, parity p taking the epoch in `epochs` whose parity is p (else epochs[0])."""
        P = self.lay.parity // 4
        for q in range(self.world):
            w = self.w32(q).view(-1, 2)
            w[:, 0] = s32(PEER_WORD[0])
            w[:, 1] = s32(PEER_WORD[1])
            if q in polled:
                for p in (0, 1):
                    e = next((e for e in epochs if (e & 1) == p), epochs[0])
                    blk = self.w32(q)[p * P:(p + 1) * P].view(-1, 2)
                    blk[:, 0] = s32(poison)
                    blk[:, 1] = s32(e)
            self.set_counter(q, counter, 0)
        for q in range(self.world):
            assert self.counter(q) == (counter, 0)

    def set_counter(self, q, counter, ticket):
        self.w32(q)[self.lay.counter // 4:self.lay.counter // 4 + 2] = i32([counter, ticket])

    def counter(self, q):
        c = self.w32(q)[self.lay.counter // 4:self.lay.counter // 4 + 2].cpu().numpy().view(np.uint32)
        return int(c[0]), int(c[1])

    def write(self, q, words, epoch, target=None):
        """Write LL words (offsets, data) with flag `epoch` into region q (or into `target`, a copy of it)."""
        off, data = words
        if not len(off):
            return
        w = self.w32(q) if target is None else target.view(torch.int32)
        idx = torch.from_numpy(np.asarray(off, np.int64) // 4).to(dev)
        w[idx] = i32(data)
        w[idx + 1] = s32(epoch)

    def snapshot(self):
        return [b.clone() for b in self.buf]

    def expect(self, before, pushes, epoch, counters=None):
        """before + the words in pushes {dst: (off, data)} with flag epoch; counters {rank: (counter, ticket)}."""
        exp = [b.clone() for b in before]
        for q, words in pushes.items():
            self.write(q, words, epoch, target=exp[q])
        for q, (c, t) in (counters or {}).items():
            exp[q].view(torch.int32)[self.lay.counter // 4:self.lay.counter // 4 + 2] = i32([c, t])
        return exp

    def check(self, exp, what):
        for q in range(self.world):
            if not torch.equal(self.buf[q], exp[q]):
                d = torch.nonzero(self.buf[q] != exp[q]).flatten()
                raise AssertionError(f"{what}: region {q} differs from the model's write map at {d.numel()} bytes, first "
                                     f"offsets {d[:6].tolist()} (parity {self.lay.parity}, area {self.lay.area}, src "
                                     f"{self.lay.src})")

    def check_flags(self, q, epochs):
        """Rule 2: every word of both parities of region q still carries its parity's epoch."""
        P = self.lay.parity // 4
        for p in (0, 1):
            e = next((e for e in epochs if (e & 1) == p), epochs[0])
            flags = self.w32(q)[p * P:(p + 1) * P].view(-1, 2)[:, 1]
            bad = int((flags != s32(e)).sum().item())
            assert bad == 0, f"region {q} parity {p}: {bad} words lost the epoch flag before the polling launch (not launched)"


# ---------------------------------------------------------------------------------------------- all-reduce
def allreduce_call(regs, inp, out, nbytes, bf, rank):
    _lib.check(lib().b200_peer_allreduce(inp.data_ptr(), out.data_ptr(), nbytes, int(bf), regs.ptrs, regs.max_msg, 0, rank,
                                         regs.world, stream()), "b200_peer_allreduce")


class AllReduce:
    """One all-reduce over W ranks' contributions: the model's words per epoch parity, and rank r's launch and checks."""

    def __init__(self, world, n16, dtype, forced, seed):
        self.world, self.n16, self.dtype, self.bf = world, n16, dtype, dtype == torch.bfloat16
        self.two_shot = po.allreduce_two_shot(n16, world, forced)
        self.contrib = po.crafted_order_input(world, n16 * 8, self.bf, seed)
        self.red = po.sum_in_rank_order(self.contrib, self.bf)
        self._pushes = {}

    def pushes(self, lay, epoch):
        key = epoch & 1
        if key not in self._pushes:
            self._pushes[key] = {s: po.allreduce_pushes(lay, s, self.world, epoch, po.words_of(self.contrib[s]),
                                                        po.words_of(self.red), self.two_shot) for s in range(self.world)}
        return self._pushes[key]

    max_msg = property(lambda self: self.n16 * 16)
    poison = po.POISON_SUM

    def fill(self, regs, rank, epoch):
        regs.write(rank, po.polled_by(self.pushes(regs.lay, epoch), rank), epoch)

    def launch(self, regs, rank, inplace=False):
        """Launch rank's call (its region already filled); returns (every tensor the launch uses, its outputs)."""
        inp = dev_bits(self.contrib[rank], self.dtype)
        out = inp if inplace else sentinel((self.n16 * 8,), self.dtype)
        allreduce_call(regs, inp, out, self.n16 * 16, self.bf, rank)
        return (inp, out), [out]

    def ok(self, outs):
        return np.array_equal(bits_of(outs[0]), self.red)


# (world, n16, max_msg or None = the message, B200_AR_TWOSHOT or None, in == out)
AR_CASES = [
    (2, 1, None, None, False), (3, 1, 4096, None, False), (8, 1, None, None, False),         # 16 B (W 3 / 8: one-shot)
    (2, 511, None, None, False), (2, 512, None, None, False), (2, 513, 1 << 16, None, False),  # one-shot CTA boundary
    (4, 511, None, None, False), (4, 512, None, None, False), (4, 513, None, None, False),
    (4, 512, None, "0", False), (2, 1024, None, "1", False), (3, 513, None, "0", False),
    (3, 3 * 256, None, None, False), (3, 3 * 257, None, None, False), (8, 8 * 255, None, None, False),   # slices at 256
    (8, 8 * 257, None, None, False), (4, 4 * 513, None, None, True), (8, 8 * 257, None, "0", False),
    (2, 32768, None, None, False), (8, 32768, 1 << 20, None, False), (4, 32768, None, "0", False),   # 64-CTA cap
    (2, 65536, 1 << 20, None, False), (4, 65536, 1 << 20, "1", False), (8, 65536, 1 << 20, "0", False),
    (2, 1000, None, None, True), (3, 999, None, "0", True), (8, 2048, None, None, True),        # in == out
]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("world,n16,max_msg,forced,inplace", AR_CASES)
def test_allreduce_rank_by_rank(world, n16, max_msg, forced, inplace, dtype, monkeypatch):
    """Every rank's output has the bits of the fp32 rank-order sum rounded once (element 0 of the data cancels 2^15 against
    -2^15 before the small terms: any other order changes it), and its pushes are the model's one-shot or two-shot words."""
    if forced is not None:
        monkeypatch.setenv("B200_AR_TWOSHOT", forced)
    else:
        monkeypatch.delenv("B200_AR_TWOSHOT", raising=False)
    ar = AllReduce(world, n16, dtype, forced, seed=n16 + world)
    regs = Regions(world, max_msg or n16 * 16)
    for r in range(world):
        counter = 1000 + r                        # both parities across the ranks
        epoch = counter + 1
        regs.prefill(counter, {r}, [epoch], po.POISON_SUM)
        ar.fill(regs, r, epoch)
        before = regs.snapshot()
        _, outs = ar.launch(regs, r, inplace)
        torch.cuda.synchronize()
        assert ar.ok(outs), f"rank {r}: all-reduce bits differ ({'two' if ar.two_shot else 'one'}-shot)"
        regs.check(regs.expect(before, ar.pushes(regs.lay, epoch)[r], epoch, {r: (epoch, 0)}), f"rank {r}")


# ---------------------------------------------------------------------------------------------- all-reduce + norm
def norm_call(regs, inp, residual, gamma, y, bf, eps, rank, pushed=False):
    fn = lib().b200_peer_gather_norm if pushed else lib().b200_peer_allreduce_norm
    rows, hidden = inp.shape
    _lib.check(fn(inp.data_ptr(), residual.data_ptr(), gamma.data_ptr(), y.data_ptr(), int(bf), rows, hidden, eps, regs.ptrs,
                  regs.max_msg, rank, regs.world, stream()), "b200_peer_gather_norm" if pushed else "b200_peer_allreduce_norm")


class AllReduceNorm:
    def __init__(self, world, rows, hidden, dtype, seed, contrib=None):
        self.world, self.rows, self.hidden, self.dtype, self.bf = world, rows, hidden, dtype, dtype == torch.bfloat16
        rng = np.random.default_rng(seed)
        if contrib is None:
            scale = np.where(np.arange(rows) % 3 == 1, 1e-3, 1.0)[None, :, None]
            c = orc.round_t(rng.standard_normal((world, rows, hidden)) * scale, self.bf)
            if not self.bf:                       # fp16: the residual sum of row 0's first 8 entries overflows
                c[:, 0, :8] = orc.round_t(40000.0 / world, False)
            contrib = orc.f64_to_bits(c, self.bf)
        self.contrib = contrib
        r = orc.round_t(rng.standard_normal((rows, hidden)), self.bf)
        if not self.bf:
            r[0, :8] = 36000.0
        self.res = orc.f64_to_bits(r, self.bf)
        self.gamma = orc.f64_to_bits(orc.round_t(rng.uniform(0.5, 1.5, hidden), self.bf), self.bf)
        self.eps = 1e-5 if seed % 2 else 1e-6
        self.red, self.stored, self.y_ref, self.A = po.allreduce_norm_ref(contrib, self.res, self.gamma, self.eps, self.bf)
        self._pushes = {}

    def pushes(self, lay, epoch, pushed=False):
        key = (epoch & 1, pushed)
        if key not in self._pushes:
            self._pushes[key] = {s: po.norm_pushes(lay, s, self.world, epoch, self.contrib[s], self.red, pushed)
                                 for s in range(self.world)}
        return self._pushes[key]

    max_msg = property(lambda self: self.rows * self.hidden * 2)
    poison = po.POISON_SUM

    def fill(self, regs, rank, epoch, pushed=False):
        regs.write(rank, po.polled_by(self.pushes(regs.lay, epoch, pushed), rank), epoch)

    def tensors(self, rank, inp=None):
        inp = dev_bits(self.contrib[rank], self.dtype) if inp is None else inp
        return inp, dev_bits(self.res, self.dtype), dev_bits(self.gamma, self.dtype), sentinel((self.rows, self.hidden), self.dtype)

    def launch(self, regs, rank, inp=None, pushed=False):
        t = self.tensors(rank, inp)
        norm_call(regs, *t, self.bf, self.eps, rank, pushed)
        return t, [t[1], t[3]]

    def ok(self, outs):
        yv = orc.from_bits(bits_of(outs[1]), self.bf).astype(np.float64)
        budget = orc.norm_error_budget(self.y_ref, self.A, po.norm_chain(self.hidden), self.bf)
        return np.array_equal(bits_of(outs[0]), self.stored) and bool((np.abs(yv - self.y_ref) <= budget).all())

    def check_outputs(self, residual, y, what):
        stored = bits_of(residual)
        assert np.array_equal(stored, self.stored), \
            f"{what}: stored residual is not round_T(float(round_T(sum)) + residual) at {int((stored != self.stored).sum())} elements"
        if not self.bf:
            assert np.isinf(orc.from_bits(stored[0, :8], False)).all() and torch.isfinite(y.float()).all()
        budget = orc.norm_error_budget(self.y_ref, self.A, po.norm_chain(self.hidden), self.bf)
        budget_report(what, bits_of(y), self.y_ref, budget, NORM_FRAC, self.dtype)


def _hidden_odd(world):
    """A hidden size whose per-rank slice Cs is not a multiple of 256 and crosses the 256-thread stride."""
    return {2: 8 * 2 * 257, 4: 8 * 4 * 130, 8: 8 * 8 * 97}[world]


NORM_SHAPES = [(1, 1024), (1, 8192), (5, 4096), (5, "odd"), (32, 1024), (32, 8192), (300, 4096), (300, "odd")]
NORM_CASES = [(w, rows, h) for w in (2, 4, 8) for rows, h in NORM_SHAPES]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("world,rows,hidden", NORM_CASES)
def test_allreduce_norm_rank_by_rank(world, rows, hidden, dtype):
    """Every rank: the stored residual is round_T(float(round_T(sum)) + residual) bit for bit (inf where an fp16 row
    overflows), y is the float64 RMSNorm of the unrounded x within oracle.norm_error_budget (this kernel's chain) and the
    glue suite's rounded fractions, with the same bits on every rank; the pushes are the model's scatter and all-gather."""
    hidden = _hidden_odd(world) if hidden == "odd" else hidden
    arn = AllReduceNorm(world, rows, hidden, dtype, seed=rows * hidden + world)
    regs = Regions(world, rows * hidden * 2)
    y0 = None
    for r in range(world):
        counter = 77 + r
        epoch = counter + 1
        regs.prefill(counter, {r}, [epoch], po.POISON_SUM)
        arn.fill(regs, r, epoch)
        before = regs.snapshot()
        _, (res, y) = arn.launch(regs, r)
        torch.cuda.synchronize()
        if y0 is None:
            arn.check_outputs(res, y, f"allreduce_norm W{world} rank {r}")
            y0 = bits_of(y)
        else:
            assert np.array_equal(bits_of(res), arn.stored), f"rank {r}: stored residual differs"
            assert np.array_equal(bits_of(y), y0), f"rank {r}: y differs from rank 0's bits"
        regs.check(regs.expect(before, arn.pushes(regs.lay, epoch)[r], epoch, {r: (epoch, 0)}), f"rank {r}")


# ---------------------------------------------------------------------------------------------- reduce-scatter GEMM
FMTS = ["int4", "int8", "int8g", "f16"]
FMT_CODE = {"f16": _lib.B200_FMT_F16, "int8": _lib.B200_FMT_INT8, "int4": _lib.B200_FMT_INT4, "int8g": _lib.B200_FMT_INT8G}
BATCHES = [1, 5, 16, 17, 32, 33, 64, 100, 128]


def _rs_cases():
    """Every (format, forced split) pair once, the batches, worlds, N, bias and PDL cycling through it. Forced split s >= 2
    runs 2s - 1 k-blocks (kb / split = 2 for all but the last split, which takes 1: an uneven plan of s splits); split 1 is
    the unsplit plan (the direct epilogue); three more cases ask for more splits than the plan can give (clamped)."""
    cases = []
    for i, (fmt, split) in enumerate(itertools.product(FMTS, range(1, 9))):
        B, world = BATCHES[i % 9], (2, 4, 8)[i % 3]
        N = 1024 if B * world >= 256 else (1024, 2048, 4096)[(i // 3) % 3]
        kb = 4 if split == 1 else 2 * split - 1
        cases.append((fmt, B, world, N, kb, split, bool(i % 2), bool((i // 2) % 2)))
    cases += [("int4", 33, 4, 2048, 4, 8, True, False),     # 8 asked, 4 k-blocks: 4 splits
              ("int8g", 17, 8, 1024, 8, 7, False, True),    # 7 asked, 8 k-blocks: 2 per split, 4 splits
              ("f16", 100, 2, 1024, 3, 6, True, True)]      # 6 asked, 3 k-blocks: 3 splits
    return cases


def expected_split(kb, forced):
    s = min(forced, kb, 8)
    kbp = -(-kb // s)
    return -(-kb // kbp)


def rs_gemm_call(regs, w, x, bias, y, rank, pdl):
    B, K = x.shape
    _lib.check(lib().b200_wo_gemm_rs(w.fmt, int(x.dtype == torch.bfloat16), x.data_ptr(), B, K, w.N, w.data.data_ptr(),
                                     None if w.col_scale is None else w.col_scale.data_ptr(),
                                     None if bias is None else bias.data_ptr(), y.data_ptr(), None, 0,
                                     _lib.B200_GEMM_PDL if pdl else 0, regs.ptrs, regs.max_msg, rank, regs.world, stream()),
               "b200_wo_gemm_rs")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("fmt,B,world,N,kb,split,with_bias,pdl", _rs_cases())
def test_rs_gemm_then_gather_norm(fmt, B, world, N, kb, split, with_bias, pdl, dtype, monkeypatch):
    """All W ranks' b200_wo_gemm_rs run for real into the shared regions, one after another. Each: the owned columns of y
    have the bits of b200_wo_gemm on the same inputs, the others keep the sentinel; every pushed word is the plain GEMM's
    bits for its (row, column pair) with flag counter + 1 at the model's slot, nothing else changes, the counter does not
    move; the plain GEMM is within oracle.gemm_error_budget of float64. Then each rank's b200_peer_gather_norm, over the
    genuine words the GEMMs left in its region, gives the bits of b200_peer_allreduce_norm on the plain GEMM outputs."""
    monkeypatch.setenv("B200_GEMM_SPLITK", str(split))
    bf = dtype == torch.bfloat16
    K = kb * 128
    ns, _ = plan(K, N)
    assert ns == expected_split(kb, split), f"plan: {ns} splits"
    rng = np.random.default_rng(B * 1000 + N + kb)
    host, wd, cscale = make_weight(fmt, K, N, bf, rng)
    w = pack(fmt, host, dtype)
    assert w.fmt == FMT_CODE[fmt]
    bias = dev_bits(orc.f64_to_bits(rng.standard_normal(N), bf), dtype) if with_bias else None
    xs = [orc.round_t(rng.standard_normal((B, K)) * 0.5, bf) for _ in range(world)]
    xd = [dev_bits(orc.f64_to_bits(x, bf), dtype) for x in xs]
    ws = ops.gemm_workspace(B, [(K, N)], dev)
    plain = [ops.wo_gemm(x, w, ws, bias=bias, pdl=pdl) for x in xd]
    torch.cuda.synchronize()
    P = np.stack([bits_of(p) for p in plain])                                  # [W, B, N]
    ref, A = orc.gemm_np(np.concatenate(xs), wd, cscale, None if bias is None else orc.from_bits(bits_of(bias), bf))
    got = orc.from_bits(P.reshape(world * B, N), bf).astype(np.float64)
    ratio = np.abs(got - ref) / orc.gemm_error_budget(ref, A, K, ns, bf)
    eq, one = orc.gemm_rounded_fractions(P.reshape(world * B, N), ref, bf)
    assert not (ratio > 1.0).any() and not np.isnan(ratio).any(), f"plain GEMM outside the budget: worst {np.nanmax(ratio):.3g}"
    assert eq >= orc.GEMM_MIN_ROUNDED and one >= orc.GEMM_MIN_WITHIN_ONE, f"rounded / within one {eq:.4f} / {one:.5f}"

    regs = Regions(world, B * N * 2)
    counter = 0xFFFFFFFF if split % 2 else 41                 # epoch 0 (the wrap) on half the cases
    epoch = (counter + 1) & 0xFFFFFFFF
    regs.prefill(counter, set(range(world)), [epoch], po.POISON_SUM)
    ys = []
    for q in range(world):
        y = sentinel((B, N), dtype)
        before = regs.snapshot()
        rs_gemm_call(regs, w, xd[q], bias, y, q, pdl)
        torch.cuda.synchronize()
        yb = bits_of(y)
        own = po.owned_columns(N, world, q)
        assert np.array_equal(yb[:, own], P[q][:, own]), f"rank {q}: owned columns differ from b200_wo_gemm"
        rest = np.ones(N, bool)
        rest[own] = False
        assert (yb[:, rest] == SENTINEL).all(), f"rank {q}: {int((yb[:, rest] != SENTINEL).sum())} non-owned outputs written"
        regs.check(regs.expect(before, po.rs_gemm_pushes(regs.lay, q, world, epoch, P[q]), epoch), f"rs gemm rank {q}")
        ys.append(y)
    for q in range(world):
        assert regs.counter(q) == (counter, 0), f"rank {q}: the GEMM moved the counter"

    # gather + norm on the genuine words, against the unfused all-reduce + norm on the plain outputs (own regions)
    arn = AllReduceNorm(world, B, N, dtype, seed=B + N, contrib=P)
    ref_regs = Regions(world, B * N * 2)
    for r in range(world):
        arn.fill(regs, r, epoch, pushed=True)                # area 1: the peers' reduced slices
        regs.check_flags(r, [epoch])
        _, (res, y) = arn.launch(regs, r, inp=ys[r], pushed=True)
        ref_regs.prefill(counter, {r}, [epoch], po.POISON_SUM)
        arn.fill(ref_regs, r, epoch)
        _, (res2, y2) = arn.launch(ref_regs, r, inp=plain[r])
        torch.cuda.synchronize()
        assert regs.counter(r) == (epoch, 0) and ref_regs.counter(r) == (epoch, 0)
        assert torch.equal(res.view(torch.int16), res2.view(torch.int16)), f"rank {r}: gather_norm residual != allreduce_norm's"
        assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), f"rank {r}: gather_norm y != allreduce_norm's"
        assert np.array_equal(bits_of(res), arn.stored)


# ---------------------------------------------------------------------------------------------- argmax
def argmax_call(regs, logits, vocab_total, out, rank):
    rows, vloc = logits.shape
    _lib.check(lib().b200_peer_argmax(logits.data_ptr(), int(logits.dtype == torch.bfloat16), rows, vloc, vocab_total,
                                      out.data_ptr(), regs.ptrs, regs.max_msg, rank, regs.world, stream()), "b200_peer_argmax")


class Argmax:
    def __init__(self, world, rows, vloc, dtype, seed):
        self.world, self.rows, self.vloc, self.dtype, self.bf = world, rows, vloc, dtype, dtype == torch.bfloat16
        self.vtot = world * vloc - 5
        rng = np.random.default_rng(seed)
        f = orc.round_t(rng.standard_normal((rows, world * vloc)), self.bf)
        r = np.arange(rows)
        f[r % 7 == 1, :] = -np.inf                                  # -inf rows: index 0
        f[r % 7 == 2, ::3] = np.nan                                 # NaN entries never win
        f[r % 7 == 2, 4] = 50.0
        f[r % 7 == 3, self.vtot + 2] = 1e4                          # a maximum in a padded column
        f[r % 7 == 3, self.vtot - 1] = 60.0                         # the last real column wins
        b = (r % world) * vloc                                     # ties across a rank boundary (lowest index wins)
        f[r % 7 == 4, b[r % 7 == 4] + vloc - 1] = 70.0
        f[r % 7 == 4, np.minimum(b[r % 7 == 4] + vloc, self.vtot - 1)] = 70.0
        f[r % 7 == 5, 7] = f[r % 7 == 5, 9] = 80.0                  # a tie inside a rank
        f[r % 7 == 6, :] = np.nan                                  # nothing qualifies
        f[r % 7 == 6, vloc + 1] = -np.inf
        self.full = f
        self.bits = orc.f64_to_bits(f, self.bf)
        self.exp = po.argmax_np(f[:, :self.vtot])
        self.pairs = [po.argmax_local(f[:, s * vloc:(s + 1) * vloc], s, vloc, self.vtot) for s in range(world)]

    max_msg = property(lambda self: self.rows * 16)
    poison = po.POISON_ARGMAX

    def pushes(self, lay, epoch):
        return {s: po.argmax_pushes(lay, s, self.world, epoch, *self.pairs[s]) for s in range(self.world)}

    def fill(self, regs, rank, epoch):
        regs.write(rank, po.polled_by(self.pushes(regs.lay, epoch), rank), epoch)

    def launch(self, regs, rank):
        logits = dev_bits(np.ascontiguousarray(self.bits[:, rank * self.vloc:(rank + 1) * self.vloc]), self.dtype)
        out = torch.full((self.rows,), -7, dtype=torch.int32, device=dev)
        argmax_call(regs, logits, self.vtot, out, rank)
        return (logits, out), [out]

    def ok(self, outs):
        return np.array_equal(outs[0].cpu().numpy(), self.exp)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("rows", [1, 7, 300])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_argmax_rank_by_rank(world, rows, dtype):
    """Every rank's token equals b200_argmax on the concatenated [rows, vocab_total] logits, bit for bit: ties inside a rank
    and across a rank boundary, -inf rows, NaN entries, a NaN-only row and a maximum in a padded column."""
    am = Argmax(world, max(rows, 1), 1003, dtype, seed=rows * world)
    full = dev_bits(np.ascontiguousarray(am.bits[:, :am.vtot]), dtype)
    exp = ops.argmax(full).cpu().numpy()
    assert np.array_equal(exp, am.exp), "b200_argmax disagrees with the numpy contract"
    regs = Regions(world, rows * 16)
    for r in range(world):
        counter = 5 + r
        epoch = counter + 1
        regs.prefill(counter, {r}, [epoch], am.poison)
        am.fill(regs, r, epoch)
        before = regs.snapshot()
        _, (out,) = am.launch(regs, r)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), exp), f"rank {r}: tokens differ from b200_argmax"
        regs.check(regs.expect(before, am.pushes(regs.lay, epoch)[r], epoch, {r: (epoch, 0)}), f"argmax rank {r}")


# ---------------------------------------------------------------------------------------------- sequences
def _kind_call(kind, world, dtype, seed, monkeypatch):
    """One call of `kind`: ar1 / ar2 (one- / two-shot all-reduce), norm (all-reduce + norm) or argmax."""
    if kind in ("ar1", "ar2"):
        monkeypatch.setenv("B200_AR_TWOSHOT", "1" if kind == "ar2" else "0")
        return AllReduce(world, 8 * 300, dtype, "1" if kind == "ar2" else "0", seed)
    if kind == "norm":
        return AllReduceNorm(world, 5, 1024 * world, dtype, seed)
    return Argmax(world, 7, 1003, dtype, seed)


@pytest.mark.parametrize("pdl", [0, 1], ids=["pdl0", "pdl1"])
@pytest.mark.parametrize("counter", [6, 0xFFFFFFFE, 0xFFFFFFFF], ids=["c6", "c_fffffffe", "c_ffffffff"])
@pytest.mark.parametrize("kind", ["ar1", "ar2", "norm", "argmax"])
def test_two_calls_in_a_row(kind, counter, pdl, monkeypatch):
    """Two calls of rank 2 of 4, back to back: the second uses the other parity, the counter moves by 2 (through the wrap
    from 0xFFFFFFFF to 0, epoch 0 being parity 0), the ticket is 0 after each; with b200_set_pdl(1) as well."""
    world, rank = 4, 2
    calls = [_kind_call(kind, world, torch.float16, seed, monkeypatch) for seed in (1, 2)]
    regs = Regions(world, calls[0].max_msg)
    epochs = [(counter + 1) & 0xFFFFFFFF, (counter + 2) & 0xFFFFFFFF]
    regs.prefill(counter, {rank}, epochs, calls[0].poison)
    for call, e in zip(calls, epochs):
        call.fill(regs, rank, e)
    lib().b200_set_pdl(pdl)
    try:
        exp = regs.snapshot()
        for i, (call, e) in enumerate(zip(calls, epochs)):
            before = exp
            _, outs = call.launch(regs, rank)
            torch.cuda.synchronize()
            assert regs.counter(rank) == (e, 0), f"call {i}: counter / ticket {regs.counter(rank)}, expected ({e}, 0)"
            assert call.ok(outs), f"call {i}: wrong result"
            exp = regs.expect(before, call.pushes(regs.lay, e)[rank], e, {rank: (e, 0)})
            regs.check(exp, f"call {i}")
    finally:
        lib().b200_set_pdl(0)


def test_graph_of_two_allreduce_norms_replayed():
    """A CUDA graph holding two all_reduce_norm calls of rank 1 of 2, replayed 3 times; before each replay the host checks
    the counter moved by 2 with the ticket at 0, refills both parities for the next two epochs and resets the residual.
    Every replay gives the bits of the eager calls."""
    world, rank, dtype = 2, 1, torch.bfloat16
    calls = [AllReduceNorm(world, 32, 4096, dtype, seed) for seed in (3, 4)]
    regs = Regions(world, 32 * 4096 * 2)
    tens = [c.tensors(rank) for c in calls]
    res0 = [t[1].clone() for t in tens]

    def refill(counter):
        epochs = [(counter + 1) & 0xFFFFFFFF, (counter + 2) & 0xFFFFFFFF]
        regs.prefill(counter, {rank}, epochs, po.POISON_SUM)
        for c, e in zip(calls, epochs):
            c.fill(regs, rank, e)
        for t, r0 in zip(tens, res0):
            t[1].copy_(r0)
        return epochs

    def body():
        for c, (inp, res, g, y) in zip(calls, tens):
            norm_call(regs, inp, res, g, y, c.bf, c.eps, rank)

    counter = 0xFFFFFFFD
    refill(counter)
    body()                                                   # eager
    torch.cuda.synchronize()
    assert regs.counter(rank) == ((counter + 2) & 0xFFFFFFFF, 0)
    eager = [(bits_of(t[1]), bits_of(t[3])) for t in tens]
    for c, (r, y) in zip(calls, eager):
        assert np.array_equal(r, c.stored)
        c.check_outputs(dev_bits(r, dtype), dev_bits(y, dtype), "eager all_reduce_norm")
    counter = (counter + 2) & 0xFFFFFFFF
    refill(counter)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            body()
    torch.cuda.synchronize()
    assert regs.counter(rank) == (counter, 0), "capture launched a kernel"
    for it in range(3):
        if it:
            refill(counter)
        graph.replay()
        torch.cuda.synchronize()
        counter = (counter + 2) & 0xFFFFFFFF
        assert regs.counter(rank) == (counter, 0), f"replay {it}: counter / ticket {regs.counter(rank)}"
        for t, (r, y) in zip(tens, eager):
            assert np.array_equal(bits_of(t[1]), r) and np.array_equal(bits_of(t[3]), y), f"replay {it}: bits differ from eager"


@pytest.mark.parametrize("kind", ["ar2", "norm", "argmax"])
def test_call_recorded_in_a_decode_program(kind, monkeypatch):
    """The same call recorded into a decode program (kept as its own launch) gives the eager bits, the eager write map and
    moves the counter; recording launches nothing."""
    world, rank = 4, 3
    call = _kind_call(kind, world, torch.bfloat16, 9, monkeypatch)
    regs = Regions(world, call.max_msg)
    runs = []
    for use_program in (False, True):
        counter = 20
        regs.prefill(counter, {rank}, [counter + 1], call.poison)
        call.fill(regs, rank, counter + 1)
        before = regs.snapshot()
        if use_program:
            prog = ops.Program()
            with prog.record():
                keep, outs = call.launch(regs, rank)
            assert prog.num_launches == 1
            assert regs.counter(rank) == (counter, 0), "recording launched a kernel"
            prog.launch()
        else:
            keep, outs = call.launch(regs, rank)
        torch.cuda.synchronize()
        assert call.ok(outs) and regs.counter(rank) == (counter + 1, 0)
        regs.check(regs.expect(before, call.pushes(regs.lay, counter + 1)[rank], counter + 1, {rank: (counter + 1, 0)}),
                   "program" if use_program else "eager")
        runs.append([o.detach().cpu().contiguous().view(torch.uint8).numpy() for o in outs])
    assert all(np.array_equal(a, b) for a, b in zip(*runs)), "the program's outputs differ from the eager call's bits"
