#!/usr/bin/env python
"""GPU parity cases (test infrastructure: imported by tests/test_gpu_parity.py, also runnable by hand under gpurun): exercises every kernel against the oracle / the naive GPU
checkers and prints a compact diagnosis per case instead of stopping at the first failure."""
import math
import os
import sys
import time
import traceback

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8, B200_FMT_INT8G  # noqa: E402
from tests import ref_kernels as refk  # noqa: E402  (naive CUDA-core second opinion, test-only library)

dev = torch.device("cuda:0")
RESULTS = []


def report(name, ok, info=""):
    RESULTS.append((name, ok))
    print(f"[{'PASS' if ok else 'FAIL'}] {name} {info}", flush=True)


def diff_info(got, exp, rtol, atol):
    got = got.float().cpu().numpy().ravel()
    exp = np.asarray(exp, np.float32).ravel()
    err = np.abs(got - exp)
    bad = err > (atol + rtol * np.abs(exp))
    nbad = int(bad.sum()) + int(np.isnan(got).sum())
    info = f"max_abs_err={np.nanmax(err):.4g} bad={nbad}/{got.size}"
    if nbad:
        idx = np.flatnonzero(bad | np.isnan(got))[:6]
        info += " first_bad=" + ", ".join(f"{i}:{got[i]:.4g}/{exp[i]:.4g}" for i in idx)
    return nbad == 0, info


def guard(name, fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        report(name, False, f"EXC {type(e).__name__}: {e}")
        traceback.print_exc()
    torch.cuda.synchronize()


# Every kernel output goes through out= into a view of a larger buffer, between sentinel bands, so a store that runs past
# the output (a ragged last tile, the padding rows of a batch pad, a query row past the group) shows up. The sentinel is a
# NaN in fp16 and in bf16, and the view starts out filled with it too: an element the kernel never writes fails the value
# check.
GUARD_BYTES = 4096
SENTINEL = 0x7FC1


def guarded_empty(shape, dtype):
    """(buffer, view): the view is `shape` of `dtype`, 16-byte aligned, with GUARD_BYTES of sentinel on each side."""
    pad = GUARD_BYTES // 2
    buf = torch.full((2 * pad + math.prod(shape),), SENTINEL, dtype=torch.int16, device=dev)
    return buf, buf[pad:buf.numel() - pad].view(dtype).view(shape)


def report_bands(name, buf):
    pad = GUARD_BYTES // 2
    bad = int((buf[:pad] != SENTINEL).sum().item() + (buf[buf.numel() - pad:] != SENTINEL).sum().item())
    report(name + " [guard bands untouched]", bad == 0, f"{bad} sentinel elements overwritten" if bad else "")


# ---------------------------------------------------------------------------------------------- attention
def budget_info(got, ref, E, is_bf16):
    """Check against the float64 reference with oracle.attn_error_budget; the info line carries the worst err/budget."""
    got = got.float().cpu().numpy().reshape(ref.shape).astype(np.float64)
    ratio = np.abs(got - ref) / orc.attn_error_budget(ref, E, is_bf16)
    ratio[np.isnan(ratio)] = np.inf
    bad = ratio > 1.0
    info = f"worst err/budget={ratio.max():.3f} bad={int(bad.sum())}/{ratio.size}"
    if bad.any():
        idx = np.flatnonzero(bad)[:6]
        info += " first_bad=" + ", ".join(f"{i}:{got.flat[i]:.5g}/{ref.flat[i]:.5g}" for i in idx)
    return not bad.any(), info


def within_ulp(got, exp, is_bf16):
    """got (the kernel's T output) within one ulp of T of the float64 value exp."""
    got = got.float().cpu().numpy().reshape(exp.shape).astype(np.float64)
    err = np.abs(got - exp)
    bad = ~(err <= orc.ulp(exp, is_bf16))
    info = f"max_abs_err={np.nanmax(err):.4g} bad={int(bad.sum())}/{exp.size}"
    if bad.any():
        idx = np.flatnonzero(bad)[:6]
        info += " first_bad=" + ", ".join(f"{i}:{got.flat[i]:.5g}/{exp.flat[i]:.5g}" for i in idx)
    return not bad.any(), info


class env_set:
    """Set the library's test-hook environment variables for the duration of a block."""
    def __init__(self, env):
        self.env, self.old = env or {}, {}

    def __enter__(self):
        for k, v in self.env.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = str(v)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def make_attn_case(B, Hq, Hkv, T, lens, dtype, seed=0, shuffle=True, D=128):
    g = torch.Generator().manual_seed(seed)
    M = max(math.ceil(L / T) for L in lens)
    npages = sum(math.ceil(L / T) for L in lens) + 1
    pool = torch.randn(npages, 2, Hkv, T, D, generator=g).to(dtype)
    q = torch.randn(B, Hq, D, generator=g).to(dtype)
    perm = (torch.randperm(npages - 1, generator=g) + 1) if shuffle else torch.arange(1, npages)
    block_ids = torch.zeros(B, M, dtype=torch.int32)
    it = iter(perm.tolist())
    for b, L in enumerate(lens):
        for j in range(math.ceil(L / T)):
            block_ids[b, j] = next(it)
    seq = torch.tensor([L - 1 for L in lens], dtype=torch.int32)
    return q, pool, block_ids, seq


def pad_block_table(block_ids, T, max_len):
    """A max_seq_len looser than the sequences needs a page table that covers it: extra columns point at page 0."""
    M = max(block_ids.shape[1], -(-max_len // T))
    out = torch.zeros(block_ids.shape[0], M, dtype=torch.int32)
    out[:, : block_ids.shape[1]] = block_ids
    return out


def run_attn(q, pool, block_ids, seq, max_len=None, q_scale=1.0):
    """The kernel (output through out= between guard bands) and the naive GPU kernel on the same inputs."""
    max_len = max_len or int(seq.max().item()) + 1
    qd, poold, sd = q.to(dev), pool.to(dev), seq.to(dev)
    pl = ops.convert_block_table(pad_block_table(block_ids, pool.shape[3], max_len).to(dev))
    B, Hq = q.shape[0], q.shape[1]
    ws = ops.attn_workspace(B, Hq, pool.shape[2], max_len, dev)
    buf, out = guarded_empty((B, Hq * pool.shape[4]), q.dtype)
    ops.paged_decode_attn(qd, poold, pl, sd, max_len, ws, out=out, q_scale=q_scale)
    ref = refk.ref_paged_decode_attn(qd, poold, pl, sd, q_scale)
    torch.cuda.synchronize()
    return out, ref, ws, buf


def attn_vs_oracle(name, B, Hq, Hkv, T, lens, dtype=torch.float16, env=None, D=128, q_scale=1.0, max_len=None):
    """Checked against the float64 reference within the error budget; the C oracle (P rounded as the kernel does) and the
    naive GPU kernel are second opinions at the reference's rtol = atol = 1e-2 (bf16: 2e-2)."""
    def fn():
        with env_set(env):
            q, pool, block_ids, seq = make_attn_case(B, Hq, Hkv, T, lens, dtype, D=D)
            out, ref, ws, buf = run_attn(q, pool, block_ids, seq, max_len, q_scale)
            is_bf16 = dtype == torch.bfloat16
            f64, E = orc.paged_decode_attn_np(q.float().numpy(), pool.float().numpy(), block_ids.numpy(), seq.numpy(), T, q_scale,
                                              with_abs=True)
            ok, info = budget_info(out, f64, E, is_bf16)
            report(name + " [kernel vs float64, error budget]", ok, info)
            bits = lambda t: t.view(torch.int16).numpy().view(np.uint16)
            exp = orc.from_bits(orc.paged_decode_attn(bits(q), bits(pool), orc.convert_block_table(block_ids.numpy()),
                                                      seq.numpy(), Hq, Hkv, D, T, is_bf16=is_bf16, q_scale=q_scale), is_bf16)
            tol = 2e-2 if is_bf16 else 1e-2
            ok1, i1 = diff_info(ref, exp, tol, tol)
            report(name + " [ref-kernel vs oracle]", ok1, i1)
            ok2, i2 = diff_info(out, exp, tol, tol)
            report(name + " [kernel vs oracle]", ok2, i2)
            sem_clean = int(ws[: B * Hkv * 4].view(torch.int32).abs().sum().item()) == 0
            report(name + " [semaphores reset]", sem_clean)
            report_bands(name, buf)
    guard(name, fn)


def attn_vs_ref_big(name, B, Hq, Hkv, T, S, dtype=torch.float16, ragged=False):
    """BASELINE-size shapes: checked against the float64 reference within the error budget; the C oracle (well under a
    second per case with OpenMP) and the naive GPU kernel are second opinions at 1e-2."""
    def fn():
        rng = np.random.default_rng(4)
        lens = [int(x) for x in (rng.integers(S // 2, S + 1, B) if ragged else [S] * B)]
        q, pool, block_ids, seq = make_attn_case(B, Hq, Hkv, T, lens, dtype, seed=42)
        out, ref, _, buf = run_attn(q, pool, block_ids, seq, max_len=S)
        is_bf16 = dtype == torch.bfloat16
        f64, E = orc.paged_decode_attn_np(q.float().numpy(), pool.float().numpy(), block_ids.numpy(), seq.numpy(), T,
                                          with_abs=True)
        ok, info = budget_info(out, f64, E, is_bf16)
        report(name + " [kernel vs float64, error budget]", ok, info)
        bits = lambda t: t.view(torch.int16).numpy().view(np.uint16)
        exp = orc.from_bits(orc.paged_decode_attn(bits(q), bits(pool), orc.convert_block_table(block_ids.numpy()),
                                                  seq.numpy(), Hq, Hkv, 128, T, is_bf16=is_bf16), is_bf16)
        ok, info = diff_info(out, exp, 1e-2, 1e-2)
        report(name + " [kernel vs oracle]", ok, info)
        ok, info = diff_info(out, ref.float().cpu().numpy(), 1e-2, 1e-2)
        report(name + " [kernel vs ref-kernel]", ok, info)
        report_bands(name, buf)
    guard(name, fn)


def attn_position_probes(name, B, Hq, Hkv, T, lens, dtype=torch.float16, env=None, D=128, q_len=1, max_len=None):
    """Exact probes of which cache positions each query reads; they fail on any indexing error at any length.

    lens = tokens cached before the q_len new ones, so query j of sequence b sees positions 0 .. lens[b] + j. V holds small
    integers that differ by batch row, kv head, position and channel; cache slots past a sequence hold NaN.
    * Uniform scores: q = 0, so every p is 1 and every sum is exact in fp32. Each output is the mean of V over the positions
      the query sees, to within one ulp of T: a dropped or repeated token, a wrong page, kv head or batch row shows.
    * Dominant key: query head r of query j has q = 64 on channel c = j*group + r, and one key it sees has 64 there: a
      score at least 256 above every other visible key at head_dim <= 256, so every other p underflows to 0 even in fp32
      and the output is that key's V row exactly.
      The key sits at seq + j for several query tokens; for one, at position 0, the new token, the page and tile
      boundaries and the first token of a forced split, varied across heads. A key with twice that score sits at
      seq + j + 1, which query j must not see (for the last query it lies past the sequence, in the page's spare slots)."""
    def fn():
        with env_set(env):
            is_bf16 = dtype == torch.bfloat16
            g = Hq // Hkv
            assert q_len * g <= D
            total = [L + q_len for L in lens]
            npg = [-(-L // T) for L in total]
            npages = sum(npg) + 1
            rng = np.random.default_rng(len(name))
            perm = iter((rng.permutation(npages - 1) + 1).tolist())
            block_ids = torch.zeros(B, max(npg), dtype=torch.int32)
            for b in range(B):
                for j in range(npg[b]):
                    block_ids[b, j] = next(perm)
            K = np.full((npages, Hkv, T, D), np.nan, np.float32)
            V = np.full((npages, Hkv, T, D), np.nan, np.float32)
            vals, where = [], []
            for b in range(B):
                t = np.arange(npg[b] * T)                              # every slot of the sequence's pages
                pg, off = block_ids[b, t // T].numpy(), t % T
                h, c = np.arange(Hkv)[None, :, None], np.arange(D)[None, None, :]
                v = ((7 * t[:, None, None] + 13 * c + 31 * h + 57 * b) % 17 - 8).astype(np.float32)
                v[:, :, 0] = (t[:, None] + 29 * np.arange(Hkv)[None] + 53 * b) % 251 - 125
                k = rng.integers(-2, 3, v.shape).astype(np.float32)
                k[:, :, : q_len * g] = 0
                V[pg, :, off], K[pg, :, off] = v, k
                if total[b] < len(t):                                  # the first spare slot holds the last query's trap key
                    V[pg[total[b]], :, off[total[b]]], K[pg[total[b]], :, off[total[b]]] = v[total[b]], 0.0
                vals.append(v)
                where.append((pg, off))
            split = 64 * int((env or {}).get("B200_ATTN_TILES_PER_SPLIT", 0))
            target = np.zeros((B, q_len, Hkv, g), np.int64)
            for b in range(B):
                pg, off = where[b]
                last = lens[b]                                         # the new token of query 0
                for j in range(q_len):
                    for kh in range(Hkv):
                        for r in range(g):
                            c = j * g + r
                            if q_len == 1:
                                choice = [x for x in (0, last, T - 1, T, 63, 64, split) if 0 < x <= last or x == 0]
                                pos = choice[(b * Hkv * g + kh * g + r) % len(choice)]
                            else:
                                pos = last + j
                            target[b, j, kh, r] = pos
                            K[pg[pos], kh, off[pos], c] = 64.0
                            if last + j + 1 < len(pg):                   # seq + j + 1: invisible to query j
                                K[pg[last + j + 1], kh, off[last + j + 1], c] = 128.0
            pool = torch.from_numpy(np.stack([K, V], axis=1)).to(dtype)
            seq = torch.tensor(lens, dtype=torch.int32)
            ml = max_len or max(total)
            pl = ops.convert_block_table(pad_block_table(block_ids, T, ml).to(dev))
            ws = ops.attn_workspace(B * q_len, Hq, Hkv, ml, dev)

            def run(q):
                buf, out = guarded_empty((B, q_len, Hq * D), dtype)
                if q_len == 1:
                    ops.paged_decode_attn(q[:, 0].contiguous().to(dev), pool.to(dev), pl, seq.to(dev), ml, ws,
                                          out=out.view(B, Hq * D))
                else:
                    ops.paged_decode_attn_multi(q.to(dev), pool.to(dev), pl, seq.to(dev), ml, ws, out=out)
                torch.cuda.synchronize()
                return out.view(B, q_len, Hq, D), buf

            # uniform scores
            out, buf = run(torch.zeros(B, q_len, Hq, D, dtype=dtype))
            exp = np.zeros((B, q_len, Hq, D))
            for b in range(B):
                for j in range(q_len):
                    exp[b, j] = np.repeat(vals[b][: lens[b] + j + 1].astype(np.float64).mean(0), g, axis=0)
            ok, info = within_ulp(out, exp, is_bf16)
            report(name + " [uniform scores: mean of the visible positions]", ok, info)
            report_bands(name + " uniform", buf)

            # dominant key
            q = np.zeros((B, q_len, Hq, D), np.float32)
            for j in range(q_len):
                for h in range(Hq):
                    q[:, j, h, j * g + h % g] = 64.0
            out, buf = run(torch.from_numpy(q).to(dtype))
            for b in range(B):
                for j in range(q_len):
                    for h in range(Hq):
                        exp[b, j, h] = vals[b][target[b, j, h // g, h % g], h // g]
            ok, info = within_ulp(out, exp, is_bf16)
            report(name + " [dominant key: its V row exactly]", ok, info)
            report_bands(name + " dominant", buf)
            sem_clean = int(ws[: B * Hkv * 4].view(torch.int32).abs().sum().item()) == 0
            report(name + " [semaphores reset]", sem_clean)
    guard(name, fn)


# ---------------------------------------------------------------------------------------------- GEMM
def make_w4(K, N, seed=1, simple=False):
    rng = np.random.default_rng(seed)
    qp = rng.integers(0, 256, (K, N // 2)).astype(np.uint8)
    G = K // 128
    if simple:
        s = np.ones((G, N), np.float16)
        zs = np.zeros((G, N), np.float16)
    else:
        s = (np.abs(rng.standard_normal((G, N))) * 0.01 + 1e-3).astype(np.float16)
        z = rng.integers(0, 16, (G, N))
        zs = ((8 - z).astype(np.float16) * s).astype(np.float16)
    return qp, s, zs


def make_w8g(K, N, seed=1, simple=False):
    rng = np.random.default_rng(seed)
    q = rng.integers(-128, 128, (K, N)).astype(np.int8)
    G = K // 128
    if simple:
        s, zs = np.ones((G, N), np.float16), np.zeros((G, N), np.float16)
    else:   # realistic magnitude: W' ~ 0.02 like an 8-bit GPTQ layer (range / 255 per group)
        s = (np.abs(rng.standard_normal((G, N))) * 2e-4 + 3e-4).astype(np.float16)
        z = rng.integers(0, 256, (G, N))
        zs = ((128 - z).astype(np.float32) * s.astype(np.float32)).astype(np.float16)
    return q, s, zs


def _bits16(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _f64(t, is_bf16):
    return None if t is None else orc.from_bits(_bits16(t), is_bf16).astype(np.float64)


def gemm_nsplit(K, N, program):
    """The split the budget may assume: the cluster kernel's plan (B200_GEMM_SPLITK included), 1 for the persistent kernel
    (its run plan is not exposed; 1 gives the loosest bound)."""
    if program:
        return 1
    import ctypes
    from rtp_llm_b200 import _lib
    ns, kbp = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().b200_plan_gemm_split(K, N, ctypes.byref(ns), ctypes.byref(kbp)), "b200_plan_gemm_split")
    return ns.value


def gemm_vs_f64(name, y, x, w_deq, nsplit, is_bf16, cscale=None, bias=None):
    """The primary GEMM check: every output within oracle.gemm_error_budget of the float64 reference of W' = w_deq
    (oracle.dequant_exact), and the correctly rounded fractions above their thresholds. x / cscale / bias: device tensors."""
    ref, A = orc.gemm_np(_f64(x, is_bf16), w_deq, _f64(cscale, is_bf16), _f64(bias, is_bf16))
    got = _bits16(y).reshape(ref.shape)
    gv = orc.from_bits(got, is_bf16).astype(np.float64)
    ratio = np.abs(gv - ref) / orc.gemm_error_budget(ref, A, w_deq.shape[0], nsplit, is_bf16)
    ratio[np.isnan(ratio)] = np.inf
    eq, one = orc.gemm_rounded_fractions(got, ref, is_bf16)
    bad = ratio > 1.0
    ok = not bad.any() and eq >= orc.GEMM_MIN_ROUNDED and one >= orc.GEMM_MIN_WITHIN_ONE
    info = f"worst err/budget={ratio.max():.3f} rounded={eq:.5f} within_one={one:.6f} bad={int(bad.sum())}/{ratio.size}"
    if bad.any():
        idx = np.flatnonzero(bad)[:6]
        info += " first_bad=" + ", ".join(f"{i}:{gv.flat[i]:.5g}/{ref.flat[i]:.5g}" for i in idx)
    report(name + " [kernel vs float64, error budget]", ok, info)


def silu_vs_f64(name, y, x, w_deq, nsplit, is_bf16, cscale=None):
    """The fused SiLU*mul epilogue against silu(g) u of the float64 gate / up GEMMs (w_deq in the reference column order:
    gate columns, then up), within oracle.silu_mul_budget."""
    inter = w_deq.shape[1] // 2
    xv, cs = _f64(x, is_bf16), _f64(cscale, is_bf16)
    g, Ag = orc.gemm_np(xv, w_deq[:, :inter], None if cs is None else cs[:inter])
    u, Au = orc.gemm_np(xv, w_deq[:, inter:], None if cs is None else cs[inter:])
    ref = orc.silu_mul_np(g, u)
    gv = orc.from_bits(_bits16(y).reshape(ref.shape), is_bf16).astype(np.float64)
    ratio = np.abs(gv - ref) / orc.silu_mul_budget(g, Ag, u, Au, w_deq.shape[0], nsplit, is_bf16)
    ratio[np.isnan(ratio)] = np.inf
    report(name + " [fused silu*mul vs float64, error budget]", not (ratio > 1.0).any(),
           f"worst err/budget={ratio.max():.3f} bad={int((ratio > 1.0).sum())}/{ratio.size}")


def run_gemm(name, x, w, ws, program, **kw):
    """One wo_gemm call; program=True records it into a decode program and launches that, so it runs in the persistent
    kernel (it must become the program's one fused op)."""
    if not program:
        return ops.wo_gemm(x, w, ws, **kw)
    prog = ops.Program()
    with prog.record():
        y = ops.wo_gemm(x, w, ws, **kw)
    report(name + " [recorded as one persistent-kernel op]", prog.num_ops == 1, f"num_ops={prog.num_ops}")
    prog.launch()
    torch.cuda.synchronize()
    return y


def gemm_case(name, fmt, B, K, N, dtype=torch.float16, simple=False, onehot=False, env=None, bias=False, big=False,
              program=False, ws_batch=None):
    """ws_batch: size the workspace for this batch instead of B (a smaller one makes the persistent kernel take longer runs)."""
    def fn():
        with env_set(env):
            rng = np.random.default_rng(2)
            if onehot:
                xf = np.zeros((B, K), np.float32)
                for b in range(B):
                    xf[b, (b * 37 + 5) % K] = 1.0
            else:
                xf = rng.standard_normal((B, K)).astype(np.float32)
            x = torch.from_numpy(xf).to(dtype).to(dev)
            bias_t = torch.from_numpy(rng.standard_normal(N).astype(np.float32)).to(dtype).to(dev) if bias else None
            if fmt == B200_FMT_INT4:
                qp, s, zs = make_w4(K, N, simple=simple)
                qd = torch.from_numpy(qp).to(dev)
                sd, zd = torch.from_numpy(s).to(dtype).to(dev), torch.from_numpy(zs).to(dtype).to(dev)
                w = ops.pack_w4(qd, sd, zd)
                ref = refk.ref_dequant_gemm(x, fmt, qd, sd, zd, 128, bias_t)
            elif fmt == B200_FMT_INT8G:
                q8, s, zs = make_w8g(K, N, simple=simple)
                qd = torch.from_numpy(q8).to(dev)
                sd, zd = torch.from_numpy(s).to(dtype).to(dev), torch.from_numpy(zs).to(dtype).to(dev)
                w = ops.pack_w8g(qd, sd, zd)
                ref = refk.ref_dequant_gemm(x, fmt, qd, sd, zd, 128, bias_t)
            elif fmt == B200_FMT_INT8:
                q8 = rng.integers(-128, 128, (K, N)).astype(np.int8)
                # realistic magnitude: W' ~ N(0, 0.02) like the loader's scale = amax/128 (device_impl.py:190)
                s = (np.abs(rng.standard_normal(N)) * 2e-4 + 3e-4).astype(np.float32)
                if simple:
                    s[:] = 1.0
                qd, sd = torch.from_numpy(q8).to(dev), torch.from_numpy(s).to(dtype).to(dev)
                w = ops.pack_w8(qd, sd)
                ref = refk.ref_dequant_gemm(x, fmt, qd, sd, None, 128, bias_t)
            else:
                wf = (rng.standard_normal((K, N)) * 0.05).astype(np.float32)
                wd = torch.from_numpy(wf).to(dtype).to(dev)
                w = ops.pack_f16(wd)
                ref = refk.ref_dequant_gemm(x, fmt, wd, None, None, 128, bias_t)
            ws = ops.gemm_workspace(ws_batch or B, [(K, N)], dev)
            buf, y = guarded_empty((B, N), dtype)
            run_gemm(name, x, w, ws, program, bias=bias_t, out=y)
            torch.cuda.synchronize()
            is_bf16 = dtype == torch.bfloat16
            if fmt == B200_FMT_INT4:
                w_deq = orc.dequant_exact("int4", qp, _bits16(sd), _bits16(zd), 128, is_bf16)
            elif fmt == B200_FMT_INT8G:
                w_deq = orc.dequant_exact("int8g", q8, _bits16(sd), _bits16(zd), 128, is_bf16)
            elif fmt == B200_FMT_INT8:
                w_deq = orc.dequant_exact("int8", q8)
            else:
                w_deq = orc.dequant_exact("f16", _bits16(wd), is_bf16=is_bf16)
            gemm_vs_f64(name, y, x, w_deq, gemm_nsplit(K, N, program), is_bf16,
                        cscale=sd if fmt == B200_FMT_INT8 else None, bias=bias_t)
            # second opinions: the naive GPU kernel and the C oracle, at the reference's tolerance
            tol = 2e-2 if fmt == B200_FMT_INT4 else 1e-2
            if dtype == torch.bfloat16:
                tol = 4e-2
            ok, info = diff_info(y, ref.float().cpu().numpy(), tol, tol * (1 if not simple else 1))
            report(name + " [kernel vs ref-kernel]", ok, info)
            if not onehot:     # every size, BASELINE shapes included: the CPU oracle is the checker
                bits = lambda t: t.cpu().view(torch.int16).numpy().view(np.uint16)
                is_bf16 = dtype == torch.bfloat16
                if fmt == B200_FMT_INT4:
                    exp = orc.dequant_gemm(bits(x), "int4", qp, scales=bits(sd), zeros_x_scales=bits(zd), group=128,
                                           bias=bits(bias_t) if bias else None, is_bf16=is_bf16)
                elif fmt == B200_FMT_INT8G:
                    exp = orc.dequant_gemm(bits(x), "int8g", q8, scales=bits(sd), zeros_x_scales=bits(zd), group=128,
                                           bias=bits(bias_t) if bias else None, is_bf16=is_bf16)
                elif fmt == B200_FMT_INT8:
                    exp = orc.dequant_gemm(bits(x), "int8", q8, scales=bits(sd), bias=bits(bias_t) if bias else None,
                                           is_bf16=is_bf16)
                else:
                    exp = orc.dequant_gemm(bits(x), "f16", bits(wd), bias=bits(bias_t) if bias else None, is_bf16=is_bf16)
                ok2, i2 = diff_info(y, orc.from_bits(exp, is_bf16), tol, tol)
                report(name + " [kernel vs oracle]", ok2, i2)
            sem_clean = int(ws[:16384].view(torch.int32).abs().sum().item()) == 0
            report(name + " [semaphores reset]", sem_clean)
            report_bands(name, buf)
    guard(name, fn)


def gemm_silu_case(name, fmt, B, K, inter, dtype=torch.float16, env=None, program=False):
    """w13 GEMM with the fused SiLU*mul epilogue against silu(g) u of the float64 GEMM within oracle.silu_mul_budget, and
    the C oracle (GEMM on the un-permuted weight, then silu_and_mul) as a second opinion."""
    def fn():
        with env_set(env):
            rng = np.random.default_rng(9)
            N = 2 * inter
            x = torch.from_numpy(rng.standard_normal((B, K)).astype(np.float32)).to(dtype).to(dev)
            bits = lambda t: t.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
            if fmt == B200_FMT_INT4:
                qp, s, zs = make_w4(K, N)
                qd, sd, zd = torch.from_numpy(qp).to(dev), torch.from_numpy(s).to(dtype).to(dev), torch.from_numpy(zs).to(dtype).to(dev)
                w = ops.pack_w4(ops.interleave_gate_up(qd, inter, packed_int4=True), ops.interleave_gate_up(sd, inter),
                                ops.interleave_gate_up(zd, inter))
                gu = orc.dequant_gemm(bits(x), "int4", qp, scales=bits(sd), zeros_x_scales=bits(zd), group=128)
            elif fmt == B200_FMT_INT8G:
                q8, s, zs = make_w8g(K, N)
                qd, sd, zd = torch.from_numpy(q8).to(dev), torch.from_numpy(s).to(dtype).to(dev), torch.from_numpy(zs).to(dtype).to(dev)
                w = ops.pack_w8g(ops.interleave_gate_up(qd, inter), ops.interleave_gate_up(sd, inter), ops.interleave_gate_up(zd, inter))
                gu = orc.dequant_gemm(bits(x), "int8g", q8, scales=bits(sd), zeros_x_scales=bits(zd), group=128)
            elif fmt == B200_FMT_INT8:
                q8 = rng.integers(-128, 128, (K, N)).astype(np.int8)
                s = (np.abs(rng.standard_normal(N)) * 2e-4 + 3e-4).astype(np.float32)
                qd, sd = torch.from_numpy(q8).to(dev), torch.from_numpy(s).to(dtype).to(dev)
                w = ops.pack_w8(ops.interleave_gate_up(qd, inter), ops.interleave_gate_up(sd, inter))
                gu = orc.dequant_gemm(bits(x), "int8", q8, scales=bits(sd))
            else:
                wd = torch.from_numpy((rng.standard_normal((K, N)) * 0.05).astype(np.float32)).to(dtype).to(dev)
                w = ops.pack_f16(ops.interleave_gate_up(wd, inter))
                gu = orc.dequant_gemm(bits(x), "f16", bits(wd))
            exp = orc.from_bits(orc.silu_and_mul(gu), False)
            ws = ops.gemm_workspace(B, [(K, N)], dev)
            buf, y = guarded_empty((B, inter), dtype)
            run_gemm(name, x, w, ws, program, silu_mul=True, out=y)
            torch.cuda.synchronize()
            is_bf16 = dtype == torch.bfloat16
            if fmt == B200_FMT_INT4:
                w_deq = orc.dequant_exact("int4", qp, bits(sd), bits(zd), 128, is_bf16)
            elif fmt == B200_FMT_INT8G:
                w_deq = orc.dequant_exact("int8g", q8, bits(sd), bits(zd), 128, is_bf16)
            elif fmt == B200_FMT_INT8:
                w_deq = orc.dequant_exact("int8", q8)
            else:
                w_deq = orc.dequant_exact("f16", bits(wd), is_bf16=is_bf16)
            silu_vs_f64(name, y, x, w_deq, gemm_nsplit(K, N, program), is_bf16, cscale=sd if fmt == B200_FMT_INT8 else None)
            ok, info = diff_info(y, exp, 2e-2, 2e-2)
            report(name + " [fused silu*mul vs oracle]", ok, info)
            report_bands(name, buf)
    guard(name, fn)


def glue_cases():
    def fn():
        rng = np.random.default_rng(3)
        for dtype in (torch.float16, torch.bfloat16):
            is_bf16 = dtype == torch.bfloat16
            bits = lambda t: t.cpu().view(torch.int16).numpy().view(np.uint16)
            x = torch.from_numpy(rng.standard_normal((5, 4096)).astype(np.float32)).to(dtype).to(dev)
            r = torch.from_numpy(rng.standard_normal((5, 4096)).astype(np.float32)).to(dtype).to(dev)
            gmm = torch.from_numpy(rng.standard_normal(4096).astype(np.float32)).to(dtype).to(dev)
            r2 = r.clone()
            y = ops.add_rmsnorm(x, r2, gmm, 1e-6)
            ye, re_ = orc.add_rmsnorm(bits(x), bits(r), bits(gmm), 1e-6, is_bf16)
            ok, info = diff_info(y, orc.from_bits(ye, is_bf16), 2e-2, 2e-2)
            report(f"add_rmsnorm {dtype}", ok and bool((bits(r2) == re_).all()), info)
            gu = torch.from_numpy(rng.standard_normal((5, 2 * 1024)).astype(np.float32)).to(dtype).to(dev)
            s = ops.silu_and_mul(gu)
            ok, info = diff_info(s, orc.from_bits(orc.silu_and_mul(bits(gu), is_bf16), is_bf16), 2e-2, 2e-2)
            report(f"silu_and_mul {dtype}", ok, info)
            B, Hq, Hkv, D, T, M = 3, 8, 2, 128, 16, 4
            qkv = torch.from_numpy(rng.standard_normal((B, (Hq + 2 * Hkv) * D)).astype(np.float32)).to(dtype).to(dev)
            pool = torch.zeros(1 + B * M, 2, Hkv, T, D, dtype=dtype, device=dev)
            block_ids = (torch.arange(B * M, dtype=torch.int32) + 1).reshape(B, M).to(dev)
            pl = ops.convert_block_table(block_ids)
            seq = torch.tensor([0, 37, 63], dtype=torch.int32, device=dev)
            qo = ops.rope_append(qkv, pool, pl, seq, Hq, 500000.0)
            qe, poole = orc.rope_append(bits(qkv), bits(torch.zeros_like(pool)), pl.cpu().numpy(), seq.cpu().numpy(), Hq,
                                        Hkv, D, T, 500000.0, is_bf16)
            ok1, i1 = diff_info(qo, orc.from_bits(qe, is_bf16), 2e-2, 2e-2)
            ok2, i2 = diff_info(pool, orc.from_bits(poole, is_bf16), 2e-2, 2e-2)
            report(f"rope_append {dtype}", ok1 and ok2, i1 + " | " + i2)
        lg = torch.randn(7, 128256, device=dev)
        lg[2, 10] = lg[2, 500] = 99.0
        am = ops.argmax(lg)
        report("argmax fp32", bool((am.cpu().numpy() == orc.argmax(lg.cpu().numpy())).all()))
        for dt in (torch.float16, torch.bfloat16):
            lh = lg.to(dt)                                   # rounding creates many exact ties: lowest index must win
            ah = ops.argmax(lh)
            report(f"argmax {dt} (vectorised path, ties)", bool((ah.cpu().numpy() == orc.argmax(lh.float().cpu().numpy())).all()))
            lo = lh[:, :1001].contiguous()                   # vocab % 8 != 0 -> scalar path
            report(f"argmax {dt} (scalar path)", bool((ops.argmax(lo).cpu().numpy() == orc.argmax(lo.float().cpu().numpy())).all()))
        tbl = torch.randn(1000, 4096, device=dev).half()
        ids = torch.tensor([3, 999, 0], dtype=torch.int32, device=dev)
        report("embedding", bool((ops.embedding(ids, tbl) == tbl[ids.long()]).all()))
        bid = torch.randint(0, 512, (4, 8), dtype=torch.int32)
        plan = ops.paged_attn_plan(torch.tensor([9, 19, 64, 129], dtype=torch.int32, device=dev),
                                   torch.arange(4 * 9, dtype=torch.int32).reshape(4, 9).to(dev), 16)
        pe = orc.paged_attn_plan(np.array([9, 19, 64, 129], np.int32), np.arange(36, dtype=np.int32).reshape(4, 9), 16)
        ok = all(np.array_equal(plan[k].cpu().numpy()[: len(pe[k])], pe[k]) for k in pe)
        report("paged_attn_plan", ok)
        report("convert_block_table", np.array_equal(ops.convert_block_table(bid.to(dev)).cpu().numpy(),
                                                     orc.convert_block_table(bid.numpy())))
    guard("glue", fn)


if __name__ == "__main__":
    which = sys.argv[1:] or ["attn", "gemm", "glue"]
    ops.device_check(0)
    print(torch.cuda.get_device_name(0), flush=True)
    t0 = time.time()
    if "glue" in which:
        glue_cases()
    if "attn" in which:
        attn_vs_oracle("attn B1 len1 p64 g4", 1, 4, 1, 64, [1])
        attn_vs_oracle("attn B2 p64 g4 [10,64]", 2, 8, 2, 64, [10, 64])
        attn_vs_oracle("attn B4 p64 g4 [65,128,200,513]", 4, 8, 2, 64, [65, 128, 200, 513])
        attn_vs_oracle("attn p16 g4", 4, 8, 2, 16, [10, 20, 65, 130])
        attn_vs_oracle("attn p32 mha", 3, 4, 4, 32, [64, 65, 1])
        attn_vs_oracle("attn p128 g8", 3, 16, 2, 128, [127, 129, 300])
        attn_vs_oracle("attn p64 g16", 2, 16, 1, 64, [100, 257])
        attn_vs_oracle("attn p64 g4 bf16", 3, 8, 2, 64, [63, 64, 300], dtype=torch.bfloat16)
        attn_vs_oracle("attn forced split 1 tile", 3, 8, 2, 64, [63, 64, 700], env={"B200_ATTN_TILES_PER_SPLIT": 1})
        attn_vs_oracle("attn forced nosplit", 3, 8, 2, 64, [63, 64, 700], env={"B200_ATTN_TILES_PER_SPLIT": 1000})
        attn_vs_ref_big("attn Llama B32 S2048", 32, 32, 8, 64, 2048)
        attn_vs_ref_big("attn Llama B32 S2048 ragged", 32, 32, 8, 64, 2048, ragged=True)
        attn_vs_ref_big("attn Qwen72B-TP8 B16 S8192", 16, 8, 1, 64, 8192)
    fmts = [(f, n) for f, n in ((B200_FMT_F16, "f16"), (B200_FMT_INT8, "int8"), (B200_FMT_INT4, "int4"))
            if "gemm" in which or f"gemm:{n}" in which]
    if fmts:
        for fmt, nm in fmts:
            gemm_case(f"gemm {nm} onehot simple B16 K128 N128", fmt, 16, 128, 128, simple=True, onehot=True)
            gemm_case(f"gemm {nm} simple B16 K128 N128", fmt, 16, 128, 128, simple=True)
            gemm_case(f"gemm {nm} B16 K256 N256", fmt, 16, 256, 256)
            gemm_case(f"gemm {nm} B5 K512 N384 bias", fmt, 5, 512, 384, bias=True)
            gemm_case(f"gemm {nm} B32 K1024 N256 splitk4", fmt, 32, 1024, 256, env={"B200_GEMM_SPLITK": 4})
            gemm_case(f"gemm {nm} B19 K1024 N384 splitk3 bias cluster", fmt, 19, 1024, 384, env={"B200_GEMM_SPLITK": 3}, bias=True)
            gemm_case(f"gemm {nm} B33 K512 N200 (ragged N, bpad64)", fmt, 33, 512, 200)
            gemm_case(f"gemm {nm} B100 K512 N256 (bpad128)", fmt, 100, 512, 256)
            gemm_case(f"gemm {nm} bf16 B8 K256 N256", fmt, 8, 256, 256, dtype=torch.bfloat16)
            gemm_silu_case(f"gemm {nm} silu B7 K256 I192", fmt, 7, 256, 192)
            gemm_silu_case(f"gemm {nm} silu B32 K1024 I128 cluster split 4", fmt, 32, 1024, 128, env={"B200_GEMM_SPLITK": 4})
    if "gemm" in which or "gemm:big" in which:
        gemm_case("gemm int4 Llama qkv B32", B200_FMT_INT4, 32, 4096, 6144, big=True)
        gemm_case("gemm int4 Llama w2 B32", B200_FMT_INT4, 32, 14336, 4096, big=True)
        gemm_case("gemm int4 Llama w13 B64", B200_FMT_INT4, 64, 4096, 28672, big=True)
        gemm_case("gemm f16 lm_head-ish B32", B200_FMT_F16, 32, 4096, 16032, big=True)
    nfail = sum(1 for _, ok in RESULTS if not ok)
    print(f"SUMMARY: {len(RESULTS) - nfail} passed, {nfail} failed, {time.time() - t0:.1f}s", flush=True)
    sys.exit(1 if nfail else 0)
