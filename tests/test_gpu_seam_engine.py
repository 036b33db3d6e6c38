"""The attention and Linear seams driven the way an engine drives them, on an H100.

  A. Where the lengths live: sequence_lengths in CUDA or in pinned host memory, through the Python B200DecodeImpl and the
     pybind B200AttnOp + b200_rope_kvcache_decode, for plain Base rope and the _ex routes (Llama3; Yarn table with
     combo_position_ids). All four runs give the same bits, the pool holds the bits of the direct rope op, and the output is
     within the float64 budget of the attention (oracle.attn_error_budget).
  B. CUDA-graph replay as an engine's graph runner does it: capture once, then each step hands prepare_cuda_graph new input
     objects (lengths grown across pages, a slot reset to a new request, block-table rows permuted and grown, new position
     ids, new qkv) and replays. Every step carries the bits of a freshly built eager impl, with PDL off and on.
  C. The engine's plan: a page table sized for a 131072-token model context, so the attention plans its split over the whole
     context. Exact position probes (uniform scores, a dominant key, NaN past each sequence) and the float64 budget for short
     sequences, where most splits are empty, and for one ~100k-token MQA sequence.
  D. B200WeightOnlyLinear at 1..1000 rows in 128-row slabs, every weight format: the float64 GEMM budget, each slab's bits
     against a direct ops.wo_gemm, graph replay, and 0 rows.
  E. Refusals: lengths a kernel cannot read (pageable host, int64, too short) and a bias or out of the wrong type or size
     raise before anything reaches the library. Pageable lengths are never handed to a forward call."""
import ctypes
import functools
import importlib.util
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import _lib, attention, build, linear, ops, rope  # noqa: E402
from rtp_llm_b200._lib import B200Error  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests.test_gpu_gemm_exact import budget_check, make_weight, plan, tdev  # noqa: E402

DEV = torch.device("cuda")
DT = {"f16": torch.float16, "bf16": torch.bfloat16}

# rope routes: plain Base runs b200_rope_append(_multi); Llama3 and the Yarn table (with position ids) run the _ex entries
ROPES = {
    "base": dict(style=1, dim=0, base=500000.0, scale=1.0),
    "llama3": dict(style=6, dim=0, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192),
    "yarn_pid": dict(style=5, dim=0, base=10000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=1024, mscale=1.13),
}


def i16(t):
    """Bit view for exact comparisons (NaN-safe)."""
    return t.contiguous().view(torch.int16)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(i16(a), i16(b))


def lengths(vals, residency):
    t = torch.tensor(vals, dtype=torch.int32)
    return t.to(DEV) if residency == "cuda" else t.pin_memory()


def position_ids(B, q_len, route, step=0):
    """combo_position_ids for the Yarn route: odd rows rotate at their own positions, even rows keep the cache slot (0)."""
    if route != "yarn_pid":
        return None
    return torch.tensor([(0 if b % 2 == 0 else 600 + 7 * b + 5 * step + j) for b in range(B) for j in range(q_len)],
                        dtype=torch.int32, device=DEV)


@functools.lru_cache(maxsize=None)
def pybind():
    spec = importlib.util.spec_from_file_location("b200_compute_ops", build.build_pybind())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.rtp_llm_ops


def py_cfg(Hq, Hkv, D, T, max_seq_len, route="base", need_rope=True):
    return SimpleNamespace(head_num=Hq, kv_head_num=Hkv, size_per_head=D, tokens_per_block=T, kernel_tokens_per_block=T,
                           max_seq_len=max_seq_len, q_scaling=1.0, need_rope_kv_cache=need_rope, use_logn_attn=False,
                           kv_cache_dtype="BASE", rope_config=SimpleNamespace(**ROPES[route]))


def py_inputs(seq, block_ids, q_len, pid=None):
    return SimpleNamespace(is_prefill=False, sequence_lengths=seq, kv_cache_kernel_block_id_device=block_ids,
                           input_lengths=torch.full((block_ids.shape[0],), q_len, dtype=torch.int32), combo_position_ids=pid)


def pb_cfg(m, Hq, Hkv, D, T, max_seq_len, route="base"):
    cfg = m.AttentionConfigs()
    cfg.head_num, cfg.kv_head_num, cfg.size_per_head, cfg.tokens_per_block, cfg.max_seq_len = Hq, Hkv, D, T, max_seq_len
    r = m.RopeConfig()
    for k, v in ROPES[route].items():
        setattr(r, k, v)
    cfg.rope_config = r
    return cfg


def pb_inputs(m, seq, block_ids, q_len, pid=None):
    inp = m.PyAttentionInputs()
    inp.sequence_lengths, inp.kv_cache_kernel_block_id_device = seq, block_ids
    inp.input_lengths = torch.full((block_ids.shape[0],), q_len, dtype=torch.int32)
    if pid is not None:
        inp.combo_position_ids = pid
    return inp


def pb_layer(m, pool):
    kv = m.LayerKVCache()
    kv.kv_cache_base = pool
    return kv


def run_python_seam(cfg, inputs, qkv, pool):
    impl = attention.B200DecodeImpl(cfg, inputs)
    return impl.forward(qkv, SimpleNamespace(kv_cache_base=pool))


def run_pybind_seam(m, cfg, inputs, qkv, pool):
    op = m.B200AttnOp(cfg)
    assert op.support(inputs)
    params = op.prepare(inputs)
    kv = pb_layer(m, pool)
    return op.forward(m.b200_rope_kvcache_decode(qkv, kv, params, cfg), kv, params)


def direct_rope(route, D, qkv, pool, block_ids, seq_cuda, Hq, q_len, pid):
    """The rope + append op called directly with CUDA lengths (the kernel is pinned in test_gpu_glue_exact)."""
    spec = rope.spec_of(SimpleNamespace(**ROPES[route]), D)
    return rope.rope_append(spec, qkv, pool, ops.convert_block_table(block_ids), seq_cuda, Hq, q_len=q_len, position_ids=pid)


def check_budget(out, q, pool, block_ids, lens, T, q_len, is_bf16, what=""):
    """out within oracle.attn_error_budget of the float64 attention of the rotated q on the appended pool."""
    B, D = len(lens), pool.shape[-1]
    qf = q.float().cpu().numpy().reshape(B, q_len, -1, D)
    ref, E = orc.paged_decode_attn_np(qf if q_len > 1 else qf[:, 0], pool.float().cpu().numpy(), block_ids.cpu().numpy(),
                                      np.asarray(lens, np.int32), T, with_abs=True)
    ok, info = probe.budget_info(out, ref, E, is_bf16)
    print(f"ATTNSTAT {what}: {info}")
    assert ok, info


def attn_case(B, q_len, Hq, Hkv, D, T, M, dtype, seed, spare_pages=0):
    """Random pool [P, 2, Hkv, T, D] with B disjoint rows of M shuffled pages, and qkv [B*q_len, (Hq+2Hkv)*D]."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = B * M + 1 + spare_pages
    pool = torch.randn(P, 2, Hkv, T, D, generator=g, device=DEV).to(dtype)
    block_ids = (torch.randperm(P - 1, generator=g, device=DEV).to(torch.int32) + 1)[:B * M].reshape(B, M).contiguous()
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    return pool, block_ids, qkv


# ---------------------------------------------------------------------------------------------- A. where the lengths live
MODEL_CTX = 256     # cfg.max_seq_len; one sequence has exactly this many tokens cached, so its new ones open a 64-token tile


@pytest.mark.parametrize("shape", [(64, 16), (128, 64), (256, 128)], ids=lambda s: f"D{s[0]}-T{s[1]}")
@pytest.mark.parametrize("q_len", [1, 3])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("route", list(ROPES))
def test_lengths_in_cuda_or_pinned_memory_give_the_same_bits_through_both_seams(route, dt, q_len, shape):
    D, T = shape
    dtype, is_bf16 = DT[dt], dt == "bf16"
    B, Hq, Hkv = 5, 8, 2
    lens = [0, T - 1, T, 2 * T - q_len, MODEL_CTX]           # empty, one short of a page, a page, ending on a page, at the bound
    M = -(-(MODEL_CTX + q_len) // T)
    pool0, block_ids, qkv = attn_case(B, q_len, Hq, Hkv, D, T, M, dtype, seed=D + T + q_len)
    pid = position_ids(B, q_len, route)
    pool_ref = pool0.clone()
    q_ref = direct_rope(route, D, qkv, pool_ref, block_ids, lengths(lens, "cuda"), Hq, q_len, pid)
    m = pybind()
    runs = {}
    for residency in ("cuda", "pinned"):
        seq = lengths(lens, residency)
        pool = pool0.clone()
        runs["python", residency] = (run_python_seam(py_cfg(Hq, Hkv, D, T, MODEL_CTX, route), py_inputs(seq, block_ids, q_len, pid),
                                                     qkv, pool), pool)
        pool = pool0.clone()
        runs["pybind", residency] = (run_pybind_seam(m, pb_cfg(m, Hq, Hkv, D, T, MODEL_CTX, route),
                                                     pb_inputs(m, seq, block_ids, q_len, pid), qkv, pool), pool)
    torch.cuda.synchronize()
    for key, (out, pool) in runs.items():
        check_budget(out, q_ref, pool_ref, block_ids, lens, T, q_len, is_bf16, f"A {key} {route} {dt} q_len {q_len} D{D} T{T}")
    out0 = runs["python", "cuda"][0]
    for key, (out, pool) in runs.items():
        assert same_bits(out, out0), f"{key}: output differs from the Python seam with CUDA lengths"
        assert same_bits(pool, pool_ref), f"{key}: pool differs from the direct rope op"


# ---------------------------------------------------------------------------------------------- B. graph replay
class Batch:
    """A batch the way an engine's scheduler moves it between steps: each sequence owns its pages, grows by q_len tokens a
    step (taking a fresh page when it crosses one), a slot can be reset to a new request, and rows change order."""

    def __init__(self, lens, T, M, P, seed):
        self.T, self.M = T, M
        self.rng = np.random.default_rng(seed)
        self.free = iter((self.rng.permutation(P - 1) + 1).tolist())
        self.lens = list(lens)
        self.pages = [[] for _ in self.lens]

    def grow(self, q_len):
        self.lens = [L + q_len for L in self.lens]

    def reset(self, slot, L):
        self.lens[slot] = L
        self.pages[slot] = []

    def rows(self, q_len, residency, route, step):
        """New input tensors for this step, rows in a new order: (lens, lengths tensor, block ids [B, M], position ids)."""
        for s, L in enumerate(self.lens):
            while len(self.pages[s]) < -(-(L + q_len) // self.T):
                self.pages[s].append(next(self.free))
        order = self.rng.permutation(len(self.lens))
        block_ids = torch.zeros(len(order), self.M, dtype=torch.int32)
        for r, s in enumerate(order):
            block_ids[r, :len(self.pages[s])] = torch.tensor(self.pages[s], dtype=torch.int32)
        lens = [self.lens[s] for s in order]
        return lens, lengths(lens, residency), block_ids.to(DEV), position_ids(len(order), q_len, route, step)


STEPS = 7


@pytest.mark.parametrize("residency", ["cuda", "pinned"])
@pytest.mark.parametrize("pdl", [False, True], ids=["pdl_off", "pdl_on"])
@pytest.mark.parametrize("route,q_len,dt", [("base", 1, "f16"), ("yarn_pid", 3, "bf16")], ids=["base-q1-f16", "yarn_pid-q3-bf16"])
def test_python_seam_graph_replay_refreshed_by_prepare_cuda_graph(route, q_len, dt, pdl, residency):
    dtype, is_bf16 = DT[dt], dt == "bf16"
    B, Hq, Hkv, D, T, M = 4, 8, 2, 128, 16, 8
    cfg = py_cfg(Hq, Hkv, D, T, 100, route)
    batch = Batch([5, 14, 31, 47], T, M, P=1 + 3 * B * M, seed=q_len)
    pool = torch.randn(1 + 3 * B * M, 2, Hkv, T, D, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV).to(dtype)
    g = torch.Generator(device=DEV).manual_seed(11)
    new_qkv = lambda: torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    lens, seq, block_ids, pid = batch.rows(q_len, residency, route, 0)
    ops.set_pdl(pdl)
    try:
        impl = attention.B200DecodeImpl(cfg, py_inputs(seq, block_ids, q_len, pid))
        qkv_in = new_qkv()
        impl.forward(qkv_in, SimpleNamespace(kv_cache_base=pool.clone()))        # loads the kernels before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out_g = impl.forward(qkv_in, SimpleNamespace(kv_cache_base=pool))
        for step in range(STEPS):
            if step == 3:
                batch.reset(2, 2)                                               # slot 2 now serves a new, short request
            if step:
                lens, seq, block_ids, pid = batch.rows(q_len, residency, route, step)
            inputs = py_inputs(seq, block_ids, q_len, pid)                      # new objects every step
            qkv = new_qkv()
            impl.prepare_cuda_graph(inputs)
            qkv_in.copy_(qkv)
            torch.cuda.synchronize()
            pool_before = pool.clone()
            graph.replay()
            torch.cuda.synchronize()
            pool_e = pool_before.clone()
            out_e = run_python_seam(cfg, inputs, qkv, pool_e)
            pool_d = pool_before.clone()
            q_d = direct_rope(route, D, qkv, pool_d, block_ids, lengths(lens, "cuda"), Hq, q_len, pid)
            torch.cuda.synchronize()
            assert same_bits(out_g, out_e), f"step {step}: replay differs from a fresh eager impl (lens {lens})"
            assert same_bits(pool, pool_e) and same_bits(pool, pool_d), f"step {step}: pool differs"
            check_budget(out_g, q_d, pool_d, block_ids, lens, T, q_len, is_bf16, f"B {route} step {step}")
            batch.grow(q_len)
    finally:
        ops.set_pdl(False)


@pytest.mark.parametrize("residency", ["cuda", "pinned"])
@pytest.mark.parametrize("pdl", [False, True], ids=["pdl_off", "pdl_on"])
@pytest.mark.parametrize("route,q_len", [("base", 1), ("yarn_pid", 3)], ids=["base-q1", "yarn_pid-q3"])
def test_pybind_seam_graph_replay_refreshed_in_place(route, q_len, pdl, residency):
    m = pybind()
    dtype = torch.float16
    B, Hq, Hkv, D, T, M = 4, 8, 2, 128, 16, 8
    cfg = pb_cfg(m, Hq, Hkv, D, T, 100, route)
    batch = Batch([3, 15, 16, 40], T, M, P=1 + 3 * B * M, seed=7 + q_len)
    pool = torch.randn(1 + 3 * B * M, 2, Hkv, T, D, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV).to(dtype)
    g = torch.Generator(device=DEV).manual_seed(13)
    new_qkv = lambda: torch.randn(B * q_len, (Hq + 2 * Hkv) * D, generator=g, device=DEV).to(dtype)
    lens, seq_cap, ids_cap, pid_cap = batch.rows(q_len, residency, route, 0)
    ops.set_pdl(pdl)
    try:
        op = m.B200AttnOp(cfg)
        params = op.prepare(pb_inputs(m, seq_cap, ids_cap, q_len, pid_cap))
        qkv_in = new_qkv()
        kv_w = pb_layer(m, pool.clone())
        op.forward(m.b200_rope_kvcache_decode(qkv_in, kv_w, params, cfg), kv_w, params)
        torch.cuda.synchronize()
        kv = pb_layer(m, pool)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out_g = op.forward(m.b200_rope_kvcache_decode(qkv_in, kv, params, cfg), kv, params)
        for step in range(STEPS):
            if step == 3:
                batch.reset(1, 1)
            if step:
                lens, seq, ids, pid = batch.rows(q_len, residency, route, step)
                seq_cap.copy_(seq)
                ids_cap.copy_(ids)
                if pid is not None:
                    pid_cap.copy_(pid)
                op.update_kv_cache_offset(params.kv_cache_offset, ids_cap)
            qkv = new_qkv()
            qkv_in.copy_(qkv)
            torch.cuda.synchronize()
            pool_e = pool.clone()
            graph.replay()
            out_e = run_pybind_seam(m, cfg, pb_inputs(m, lengths(lens, residency), ids_cap.clone(), q_len,
                                                      None if pid_cap is None else pid_cap.clone()), qkv, pool_e)
            torch.cuda.synchronize()
            assert same_bits(out_g, out_e) and same_bits(pool, pool_e), f"step {step}: replay differs from eager (lens {lens})"
            batch.grow(q_len)
    finally:
        ops.set_pdl(False)


# ---------------------------------------------------------------------------------------------- C. the engine's plan
ENGINE_CTX = 131072         # Llama-3.1's context: the page table an engine sizes for it


def attn_plan(units, max_seq_len):
    ns, tps = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.load().b200_plan_attn_split(units, max_seq_len, ctypes.byref(ns), ctypes.byref(tps)), "b200_plan_attn_split")
    return ns.value, tps.value


def engine_impl(lens, q_len, Hq, Hkv, D, T):
    """B200DecodeImpl without rope, configured for ENGINE_CTX, on a page table ENGINE_CTX / T columns wide (a sequence's
    unused columns point at page 0)."""
    cfg = py_cfg(Hq, Hkv, D, T, ENGINE_CTX, need_rope=False)
    npg = [-(-(L + q_len) // T) for L in lens]
    perm = iter((np.random.default_rng(len(lens) + q_len).permutation(sum(npg)) + 1).tolist())
    block_ids = torch.zeros(len(lens), ENGINE_CTX // T, dtype=torch.int32)
    for b, n in enumerate(npg):
        block_ids[b, :n] = torch.tensor([next(perm) for _ in range(n)], dtype=torch.int32)
    inputs = py_inputs(lengths(lens, "cuda"), block_ids.to(DEV), q_len)
    assert attention.B200DecodeImpl.support(cfg, inputs)
    return attention.B200DecodeImpl(cfg, inputs), block_ids, sum(npg) + 1


def slots(block_ids, b, n, T):
    """(page, offset) of the first n cache positions of row b."""
    t = np.arange(n)
    return block_ids[b].numpy()[t // T], t % T


def semaphores_clear(impl, B, Hkv):
    return int(impl.fmha_params.workspace[: B * Hkv * 4].view(torch.int32).abs().sum().item()) == 0


ENGINE = [("short 0", [0], 1, "f16"), ("short 64", [64], 1, "f16"), ("short 1000", [1000], 1, "bf16"),
          ("mqa 100k", [100_000], 1, "f16"), ("mqa 100k q_len 4", [99_996], 4, "bf16")]


@pytest.mark.parametrize("case", ENGINE, ids=[c[0] for c in ENGINE])
def test_attention_planned_for_the_model_context(case):
    name, lens, q_len, dt = case
    dtype, is_bf16 = DT[dt], dt == "bf16"
    B, Hkv, g, D, T = len(lens), 1, 8, 128, 64
    Hq = Hkv * g
    impl, block_ids, P = engine_impl(lens, q_len, Hq, Hkv, D, T)
    assert impl.fmha_params.max_seq_len == ENGINE_CTX
    nsplit, tps = attn_plan(B * Hkv, impl.fmha_params.max_seq_len)
    print(f"PLAN {name}: {nsplit} splits of {tps} tiles")
    assert nsplit > 32, (nsplit, tps)
    total = [L + q_len for L in lens]

    def call(pool, q):
        out = impl.forward(q.reshape(B * q_len, Hq * D).to(dtype).to(DEV).contiguous(), SimpleNamespace(kv_cache_base=pool))
        torch.cuda.synchronize()
        assert semaphores_clear(impl, B, Hkv), "workspace semaphores not back at zero"
        return out

    # exact probes, as gpu_probe.attn_position_probes builds them: V small integers, K in -2..2 with the probed channels zero,
    # NaN in every slot past a sequence (page 0 included, which the unused columns point at)
    rng = np.random.default_rng(7)
    K = np.full((P, Hkv, T, D), np.nan, np.float32)
    V = np.full((P, Hkv, T, D), np.nan, np.float32)
    vals, where = [], []
    for b in range(B):
        n = -(-total[b] // T) * T
        pg, off = slots(block_ids, b, n, T)
        t, c, h = np.arange(n)[:, None, None], np.arange(D)[None, None, :], np.arange(Hkv)[None, :, None]
        v = ((7 * t + 13 * c + 31 * h + 57 * b) % 17 - 8).astype(np.float32)
        v[:, :, 0] = (np.arange(n)[:, None] + 29 * np.arange(Hkv)[None] + 53 * b) % 251 - 125
        k = rng.integers(-2, 3, v.shape).astype(np.float32)
        k[:, :, : q_len * g] = 0
        V[pg[:total[b]], :, off[:total[b]]], K[pg[:total[b]], :, off[:total[b]]] = v[:total[b]], k[:total[b]]
        if total[b] < n:                                       # the first spare slot holds the last query's trap key
            V[pg[total[b]], :, off[total[b]]], K[pg[total[b]], :, off[total[b]]] = v[total[b]], 0.0
        vals.append(v)
        where.append((pg, off))
    target = np.zeros((B, q_len, Hkv, g), np.int64)
    for b in range(B):
        pg, off = where[b]
        last = lens[b]
        for j in range(q_len):
            for kh in range(Hkv):
                for r in range(g):
                    c = j * g + r
                    if q_len == 1:       # position 0, the new token, page and tile edges, the first tokens of splits
                        choice = [x for x in (0, last, T - 1, T, 64 * tps - 1, 64 * tps, 64 * tps * (last // (64 * tps)), last - 1)
                                  if 0 < x <= last or x == 0]
                        pos = choice[(kh * g + r) % len(choice)]
                    else:
                        pos = last + j
                    target[b, j, kh, r] = pos
                    K[pg[pos], kh, off[pos], c] = 64.0
                    if last + j + 1 < len(pg):                  # seq + j + 1: invisible to query j
                        K[pg[last + j + 1], kh, off[last + j + 1], c] = 128.0
    pool = torch.from_numpy(np.stack([K, V], axis=1)).to(dtype).to(DEV)

    out = call(pool, torch.zeros(B, q_len, Hq, D))
    exp = np.zeros((B, q_len, Hq, D))
    for b in range(B):
        for j in range(q_len):
            exp[b, j] = np.repeat(vals[b][: lens[b] + j + 1].astype(np.float64).mean(0), g, axis=0)
    ok, info = probe.within_ulp(out, exp, is_bf16)
    assert ok, "uniform scores: " + info

    q = np.zeros((B, q_len, Hq, D), np.float32)
    for j in range(q_len):
        for h in range(Hq):
            q[:, j, h, j * g + h % g] = 64.0
    out = call(pool, torch.from_numpy(q))
    for b in range(B):
        for j in range(q_len):
            for h in range(Hq):
                exp[b, j, h] = vals[b][target[b, j, h // g, h % g], h // g]
    ok, info = probe.within_ulp(out, exp, is_bf16)
    assert ok, "dominant key: " + info

    # float64 budget on random data, NaN still past each sequence
    Kr, Vr = np.full_like(K, np.nan), np.full_like(V, np.nan)
    for b in range(B):
        pg, off = where[b]
        n = total[b]
        Kr[pg[:n], :, off[:n]] = rng.standard_normal((n, Hkv, D))
        Vr[pg[:n], :, off[:n]] = rng.standard_normal((n, Hkv, D))
    pool = torch.from_numpy(np.stack([Kr, Vr], axis=1)).to(dtype)
    qr = torch.from_numpy(rng.standard_normal((B, q_len, Hq, D)).astype(np.float32)).to(dtype)
    out = call(pool.to(DEV), qr)
    qn = qr.float().numpy()
    ref, E = orc.paged_decode_attn_np(qn if q_len > 1 else qn[:, 0], pool.float().numpy(), block_ids.numpy(),
                                      np.asarray(lens, np.int32), T, with_abs=True)
    ok, info = probe.budget_info(out, ref, E, is_bf16)
    print(f"ATTNSTAT C {name}: {info}")
    assert ok, info


# ---------------------------------------------------------------------------------------------- D. Linear seam
LIN_K, LIN_N = 512, 256
ROW_SHAPES = [(1,), (2, 64), (129,), (3, 100), (4, 250)]         # 1, 128, 129, 300 and 1000 rows with leading dims
LIN_FMTS = ["int4", "int4g64", "int4g32", "int8", "int8g", "f16", "int4 act-order"]


class Q:
    def __init__(self, method):
        self.method = method

    def get_method(self):
        return self.method


def make_linear(fmt, dtype, is_bf16, bias, rng):
    """(B200WeightOnlyLinear, W' float64 [K, N] in blob row order, column scale the epilogue applies, row perm or None).
    INT8 comes as a loader hands it over: the blob without a column scale, and fp32 scales beside it."""
    K, N = LIN_K, LIN_N
    base = fmt.split()[0]
    host, wd, cscale = make_weight(base, K, N, is_bf16, rng)
    perm = rng.permutation(K) if "act-order" in fmt else None
    if base == "f16":
        return linear.B200WeightOnlyLinear(tdev(host[0], dtype), None, None, bias), wd, None, None
    if base == "int8":
        q, c = host
        c32 = torch.from_numpy(np.asarray(c * (1 + rng.uniform(-1e-3, 1e-3, N)), np.float32))   # fp32 values off the T grid
        packed = ops.PackedWeight.from_tensor(ops.pack_w8(torch.from_numpy(q).to(DEV), c32.to(DEV)).data)
        lin = linear.B200WeightOnlyLinear(packed.data, c32.to(DEV), None, bias, Q("int8"))
        return lin, wd, orc.round_t(c32.double().numpy(), is_bf16), None
    raw, s, zs = host
    sd, zd = tdev(s, dtype), tdev(zs, dtype)
    if base == "int8g":
        packed = ops.pack_w8g(torch.from_numpy(raw).to(DEV), sd, zd)
    else:
        group = {"int4": 128, "int4g64": 64, "int4g32": 32}[base]
        packed = ops.pack_w4(torch.from_numpy(raw).to(DEV), sd, zd, group,
                             perm=None if perm is None else torch.from_numpy(perm.astype(np.int32)))
    return linear.B200WeightOnlyLinear(packed.data, sd, None, bias, Q("gptq")), wd, None, perm


@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("fmt", LIN_FMTS)
def test_linear_seam_in_slabs(fmt, dt, with_bias):
    dtype, is_bf16 = DT[dt], dt == "bf16"
    K, N = LIN_K, LIN_N
    rng = np.random.default_rng(sum(map(ord, fmt + dt)) + with_bias)
    bias_np = orc.round_t(rng.standard_normal(N), is_bf16) if with_bias else None
    lin, wd, cscale, perm = make_linear(fmt, dtype, is_bf16, None if bias_np is None else tdev(bias_np, dtype), rng)
    ws = ops.gemm_workspace(lin.MAX_BATCH, [(K, N)], DEV)
    scratch = torch.empty(lin.MAX_BATCH, K, dtype=dtype, device=DEV) if perm is not None else None
    xs, ys = [], []
    for lead in ROW_SHAPES:
        x_np = orc.round_t(rng.standard_normal((int(np.prod(lead)), K)), is_bf16)
        y = lin(tdev(x_np, dtype).reshape(*lead, K))
        assert y.shape == (*lead, N) and y.dtype == dtype
        y2 = y.reshape(-1, N)
        x2 = tdev(x_np, dtype)
        for i in range(0, x2.shape[0], lin.MAX_BATCH):                   # each slab: the bits of a direct wo_gemm on it
            direct = ops.wo_gemm(x2[i:i + lin.MAX_BATCH], lin.packed, ws, bias=lin.bias, x_perm=scratch)
            assert same_bits(y2[i:i + lin.MAX_BATCH], direct), f"rows {lead}: slab at {i} differs from ops.wo_gemm"
        xs.append(x_np)
        ys.append(y2)
    x_all = np.concatenate(xs)
    ref, A = orc.gemm_np(x_all if perm is None else x_all[:, perm], wd, cscale, bias_np)
    budget_check(f"linear {fmt}", probe._bits16(torch.cat(ys)), ref, A, K, plan(K, N)[0], is_bf16, "B200WeightOnlyLinear")

    # graph replay at 300 rows on new x against the eager bits
    x_in = tdev(orc.round_t(rng.standard_normal((300, K)), is_bf16), dtype)
    lin(x_in)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g = lin(x_in)
    x_new = tdev(orc.round_t(rng.standard_normal((300, K)), is_bf16), dtype)
    x_in.copy_(x_new)
    graph.replay()
    y_e = lin(x_new)
    torch.cuda.synchronize()
    assert same_bits(y_g, y_e), "graph replay differs from eager"

    # 0 rows: an empty result, as F.linear gives, and no launch
    n0 = ops.launch_count()
    for lead in ((0,), (2, 0)):
        y0 = lin(torch.empty(*lead, K, dtype=dtype, device=DEV))
        assert y0.shape == (*lead, N) and y0.dtype == dtype
    assert ops.launch_count() == n0


# ---------------------------------------------------------------------------------------------- E. refusals
class NoLibrary:
    def __getattr__(self, name):
        pytest.fail(f"{name} was reached: the arguments should have been refused before the library")


@pytest.fixture
def forbid_library(monkeypatch):
    """install(): from then on every library entry point fails the test, so a call must be refused on the host."""
    return lambda: monkeypatch.setattr(_lib, "load", lambda: NoLibrary())


def bad_lengths(B):
    """Lengths a kernel cannot read: pageable host memory, int64, one entry short."""
    return {"pageable": torch.zeros(B, dtype=torch.int32),
            "int64": torch.zeros(B, dtype=torch.int64, device=DEV),
            "short": torch.zeros(B - 1, dtype=torch.int32, device=DEV)}


def attention_calls(seq):
    """Every attention and rope + append wrapper, with valid arguments except the lengths."""
    B, Hq, Hkv, D, T, M, dt = 4, 8, 2, 128, 16, 4, torch.float16
    pool = torch.zeros(1 + B * M, 2, Hkv, T, D, dtype=dt, device=DEV)
    pl = torch.zeros(B, 1, 2, M, dtype=torch.int32, device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    qkv = torch.zeros(B, (Hq + 2 * Hkv) * D, dtype=dt, device=DEV)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device=DEV)
    gamma = torch.ones(D, dtype=dt, device=DEV)
    cfg = rope.c_config(rope.spec_of(SimpleNamespace(**ROPES["llama3"]), D))
    q = lambda *s: torch.zeros(*s, dtype=dt, device=DEV)
    qkv2 = torch.zeros(2 * B, (Hq + 2 * Hkv) * D, dtype=dt, device=DEV)
    return {
        "paged_decode_attn": lambda: ops.paged_decode_attn(q(B, Hq, D), pool, pl, seq, M * T, ws),
        "paged_decode_attn_multi": lambda: ops.paged_decode_attn_multi(q(B, 2, Hq, D), pool, pl, seq, M * T, ws),
        "paged_decode_attn_beam": lambda: ops.paged_decode_attn_beam(q(2, 2, Hq, D), pool, pl, seq, i32(0, 0), M * T, ws),
        "paged_decode_attn_tree": lambda: ops.paged_decode_attn_tree(q(B, 2, Hq, D), pool, pl, seq, torch.zeros(B, 2, dtype=torch.int32,
                                                                                                            device=DEV), M * T, ws),
        "paged_decode_attn_rope": lambda: ops.paged_decode_attn_rope(qkv, pool, pl, seq, Hq, M * T, 10000.0, ws),
        "paged_decode_attn_prefix": lambda: ops.paged_decode_attn_prefix(q(B, Hq, D), pool, pl, seq, i32(0, 1, 2, 3, 4), i32(0, 1, 2, 3),
                                                                         i32(0, 0, 0, 0), 1, M * T, ws),
        "rope_append": lambda: ops.rope_append(qkv, pool, pl, seq, Hq, 10000.0),
        "rope_append q_len 2": lambda: ops.rope_append(qkv2, pool, pl, seq, Hq, 10000.0, q_len=2),
        "rope_append_ex q_len 2": lambda: ops.rope_append_ex(qkv2, pool, pl, seq, Hq, cfg, q_len=2),
        "rope_append_ex": lambda: ops.rope_append_ex(qkv, pool, pl, seq, Hq, cfg),
        "qk_norm_rope_append": lambda: ops.qk_norm_rope_append(qkv, gamma, gamma, 1e-6, pool, pl, seq, Hq, 10000.0),
        "qk_norm_rope_append_ex": lambda: ops.qk_norm_rope_append_ex(qkv, gamma, gamma, 1e-6, pool, pl, seq, Hq, cfg),
    }


@pytest.mark.parametrize("kind", ["pageable", "int64", "short"])
def test_attention_wrappers_refuse_unreadable_lengths(kind, forbid_library):
    B = 4
    seq = bad_lengths(B)[kind]
    forbid_library()
    for name, call in attention_calls(seq).items():
        with pytest.raises(B200Error, match="sequence_lengths"):
            call()


@pytest.mark.parametrize("kind", ["pageable", "int64", "short"])
def test_seams_refuse_unreadable_lengths_before_any_launch(kind, forbid_library):
    """B200DecodeImpl(...) and B200DecodeAttnOp.update, and the pybind prepare() / update(), refuse the lengths before they
    launch anything (neither reads lengths on the GPU). forward is never called with them."""
    B, Hq, Hkv, D, T, M = 4, 8, 2, 128, 16, 4
    block_ids = torch.arange(1, 1 + B * M, dtype=torch.int32, device=DEV).reshape(B, M)
    bad = bad_lengths(B)[kind]
    good = lengths([1, 2, 3, 4], "cuda")
    cfg = py_cfg(Hq, Hkv, D, T, M * T)
    op = attention.B200DecodeAttnOp(cfg)
    params = op.prepare(py_inputs(good, block_ids, 1))
    m = pybind()
    pcfg = pb_cfg(m, Hq, Hkv, D, T, M * T)
    pop = m.B200AttnOp(pcfg)
    pparams = pop.prepare(pb_inputs(m, good, block_ids, 1))
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="sequence_lengths"):
        pop.prepare(pb_inputs(m, bad, block_ids, 1))
    with pytest.raises(RuntimeError, match="sequence_lengths"):
        pop.update(pparams, pb_inputs(m, bad, block_ids, 1))
    assert ops.launch_count() == n0, "the pybind seam launched before refusing"
    forbid_library()
    with pytest.raises(B200Error, match="sequence_lengths"):
        attention.B200DecodeImpl(cfg, py_inputs(bad, block_ids, 1))
    with pytest.raises(B200Error, match="sequence_lengths"):
        op.update(params, py_inputs(bad, block_ids, 1))


def test_wo_gemm_and_linear_refuse_a_bias_or_out_of_the_wrong_type_or_size(forbid_library):
    K, N, B = 256, 384, 3
    f16 = dict(dtype=torch.float16, device=DEV)
    x = torch.zeros(B, K, **f16)
    w_kn = torch.zeros(K, N, **f16)
    w = ops.pack_f16(w_kn)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    lin = linear.B200WeightOnlyLinear(w_kn, None, None, torch.zeros(N, dtype=torch.float32, device=DEV))  # a loader's fp32 bias
    forbid_library()
    for bias in (torch.zeros(N, dtype=torch.float32, device=DEV), torch.zeros(N, dtype=torch.bfloat16, device=DEV),
                 torch.zeros(N - 1, **f16), torch.zeros(1, N, **f16)):
        with pytest.raises(B200Error, match="bias"):
            ops.wo_gemm(x, w, ws, bias=bias)
    for out, silu in ((torch.empty(B, N, dtype=torch.float32, device=DEV), False), (torch.empty(B, N - 128, **f16), False),
                      (torch.empty(B + 1, N, **f16), False), (torch.empty(B, N, **f16), True)):
        with pytest.raises(B200Error, match="out"):
            ops.wo_gemm(x, w, ws, out=out, silu_mul=silu)
    with pytest.raises(B200Error, match="bias"):
        lin(torch.zeros(2, 5, K, **f16))
    assert lin(torch.zeros(0, K, **f16)).shape == (0, N)                # 0 rows never reach the library
