"""The cases of tests/test_gpu_pdl_hazards.py: one per PDL entry point and path, each naming the kernels it reaches (the CPU test
test_pdl_cases.py keeps that list complete; "wo_gemm_kernel/rs" is the reduce-scatter instantiation of wo_gemm_kernel). A case's setup() runs on the GPU and returns a Spec of three groups of buffers:

- static: constant after load (packed weights, scales, bias, gammas, rope tables), built once;
- dyn(seed): every other input the call reads, as a fresh dict of device tensors per seed (0 is version A, 1.. the staged
  versions); in-place buffers are among them and named in `inplace`;
- outs: pure outputs {name: (shape, dtype)}, and ws: workspaces {name: (bytes, leading bytes of counters that must be zero
  again after a call)}, zero on entry.

call(b) launches the entry point on the current stream with b = static | dyn | outs | ws, and nothing else: no allocation
that launches a kernel, no host synchronisation."""
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np
import torch

DEV = torch.device("cuda")
F16, BF16, F32, I32 = torch.float16, torch.bfloat16, torch.float32, torch.int32
TILES, SPLITK = "B200_ATTN_TILES_PER_SPLIT", "B200_GEMM_SPLITK"


@dataclass
class Spec:
    dyn: Callable[[int], dict]
    call: Callable[[dict], None]
    static: dict = field(default_factory=dict)
    inplace: tuple = ()
    outs: dict = field(default_factory=dict)
    ws: dict = field(default_factory=dict)


@dataclass
class Case:
    name: str
    kernels: tuple
    setup: Callable[[], Spec]
    env: Optional[dict] = None
    stream: bool = True          # False: the call synchronises the host outside graph capture; graph replays only


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape, dtype=F16, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _ints(g, lo, hi, *shape):
    return torch.randint(lo, hi, shape, generator=g, dtype=I32).to(DEV)


def _page_list(g, rows, M, P):
    """A [rows, 1, 2, M] page list over distinct pages 1 .. P - 1 (rows * M * 2 <= P - 1), K and V pages apart."""
    perm = (torch.randperm(P - 1, generator=g)[: rows * 2 * M] + 1).to(I32)
    return perm.view(rows, 1, 2, M).contiguous().to(DEV)


# ---------------------------------------------------------------------------------------------- attention
def _attn(fn, dtype=F16, D=128, B=3, Hq=16, Hkv=2, T=16, q_len=1, max_len=200, W=0, chunks=()):
    """chunks (prefix): the sizes of the chunks over the B = sum(chunks) rows."""
    from rtp_llm_b200 import ops
    B = sum(chunks) or B
    rows = B * W if W else B
    M = -(-max_len // T)
    P = rows * 2 * M + 1

    def dyn(seed):
        g = _gen(seed)
        lo, hi = max(0, max_len - q_len - 64), max_len - q_len
        pl = _page_list(g, rows, M, P)
        seq = torch.randint(lo, hi + 1, (rows,), generator=g, dtype=I32)
        d = dict(pool=_randn(g, P, 2, Hkv, T, D, dtype=dtype))
        if fn == "rope":
            d["qkv"] = _randn(g, B, (Hq + 2 * Hkv) * D, dtype=dtype)
        elif fn == "beam":
            d["q"] = _randn(g, B, W, Hq, D, dtype=dtype)
            shared = torch.zeros(B, dtype=I32)
            for b in range(B):
                s = T * (int(seq[b * W: (b + 1) * W].min()) // T)
                shared[b] = s
                pl[b * W + 1: (b + 1) * W, :, :, : s // T] = pl[b * W, :, :, : s // T]
            d["shared"] = shared.to(DEV)
        elif fn == "prefix":
            # the chunk sizes in a seeded order over a seeded permutation of the rows; a chunk's members share the first
            # member's pages below their shortest cached length
            d["q"] = _randn(g, B, Hq, D, dtype=dtype)
            order = torch.randperm(B, generator=g).tolist()
            offs, shared = [0], []
            for n in (chunks[i] for i in torch.randperm(len(chunks), generator=g).tolist()):
                members = order[offs[-1]: offs[-1] + n]
                s = T * (int(seq[members].min()) // T) if n > 1 else 0
                for r in members[1:]:
                    pl[r, :, :, : s // T] = pl[members[0], :, :, : s // T]
                offs.append(offs[-1] + n)
                shared.append(s)
            d.update(offs=torch.tensor(offs, dtype=I32).to(DEV), rows=torch.tensor(order, dtype=I32).to(DEV),
                     shared=torch.tensor(shared, dtype=I32).to(DEV))
        elif fn == "single":
            d["q"] = _randn(g, B, Hq, D, dtype=dtype)
        else:
            d["q"] = _randn(g, B, q_len, Hq, D, dtype=dtype)
        if fn == "tree":
            from tests.verify_oracle import random_tree
            rng = np.random.default_rng(seed)
            d["parents"] = torch.from_numpy(np.stack([random_tree(rng, q_len, "random") for _ in range(B)])).to(I32).to(DEV)
        d.update(pl=pl, seq=seq.to(DEV))
        return d

    out_rows = (B,) if fn in ("single", "rope", "prefix") else (B, W if W else q_len)

    def call(b):
        kw = dict(out=b["out"])
        if fn == "single":
            ops.paged_decode_attn(b["q"], b["pool"], b["pl"], b["seq"], max_len, b["ws"], **kw)
        elif fn == "multi":
            ops.paged_decode_attn_multi(b["q"], b["pool"], b["pl"], b["seq"], max_len, b["ws"], **kw)
        elif fn == "beam":
            ops.paged_decode_attn_beam(b["q"], b["pool"], b["pl"], b["seq"], b["shared"], max_len, b["ws"], **kw)
        elif fn == "tree":
            ops.paged_decode_attn_tree(b["q"], b["pool"], b["pl"], b["seq"], b["parents"], max_len, b["ws"], **kw)
        elif fn == "prefix":
            ops.paged_decode_attn_prefix(b["q"], b["pool"], b["pl"], b["seq"], b["offs"], b["rows"], b["shared"], max(chunks), max_len,
                                         b["ws"], **kw)
        else:
            ops.paged_decode_attn_rope(b["qkv"], b["pool"], b["pl"], b["seq"], Hq, max_len, 10000.0, b["ws"], **kw)

    def setup():
        ws = ops.attn_workspace(rows * q_len, Hq, Hkv, max_len, DEV).numel()
        sem = -(-rows * Hkv * 4 // 256) * 256
        return Spec(dyn, call, inplace=("pool",) if fn == "rope" else (), outs={"out": ((*out_rows, Hq * D), dtype)},
                    ws={"ws": (ws, sem)})
    return setup


UNSPLIT, CLUSTER, WORKSPACE = {TILES: 64}, {TILES: 1}, {TILES: 1}
ATTN = [
    Case("attn unsplit f16", ("paged_decode_attn_kernel",), _attn("single", max_len=300), UNSPLIT),
    Case("attn cluster merge bf16", ("paged_decode_attn_kernel",), _attn("single", BF16, max_len=300), CLUSTER),
    Case("attn workspace merge f16", ("paged_decode_attn_kernel",), _attn("single", max_len=900), WORKSPACE),
    Case("attn d64 cluster merge bf16", ("paged_decode_attn_kernel",), _attn("single", BF16, D=64, Hq=8, max_len=400, T=32),
         CLUSTER),
    Case("attn d256 workspace merge f16", ("paged_decode_attn_kernel",), _attn("single", D=256, Hq=8, max_len=700, T=64),
         WORKSPACE),
    Case("attn multi rt1 f16", ("paged_decode_attn_kernel",), _attn("multi", q_len=2, Hq=16, Hkv=2, max_len=300)),
    Case("attn multi rt2 bf16", ("paged_decode_attn_kernel",), _attn("multi", BF16, q_len=4, max_len=300), CLUSTER),
    Case("attn multi rt4 f16 workspace merge", ("paged_decode_attn_kernel",), _attn("multi", q_len=8, max_len=700), WORKSPACE),
    Case("attn beam w4 bf16", ("paged_decode_attn_kernel",), _attn("beam", BF16, W=4, Hq=8, max_len=200), CLUSTER),
    Case("attn tree f16", ("paged_decode_attn_kernel",), _attn("tree", q_len=6, Hq=8, max_len=300), CLUSTER),
    Case("attn prefix chunks 3 2 1 f16 workspace merge", ("paged_decode_attn_kernel",), _attn("prefix", chunks=(3, 2, 1), max_len=600),
         WORKSPACE),
    Case("attn rope f16", ("paged_decode_attn_kernel",), _attn("rope", Hq=8, max_len=300)),
    Case("attn rope bf16 cluster merge", ("paged_decode_attn_kernel",), _attn("rope", BF16, Hq=8, max_len=300), CLUSTER),
]


# ---------------------------------------------------------------------------------------------- weight-only GEMM
def _weight(fmt, dtype, K, N, g, group=128, perm=None):
    from rtp_llm_b200 import ops
    if fmt == "int4":
        s = (torch.rand(K // group, N, generator=g) * 0.01 + 1e-3).to(dtype).to(DEV)
        qp = torch.randint(0, 256, (K, N // 2), generator=g, dtype=torch.uint8).to(DEV)
        return ops.pack_w4(qp, s, (-8 * s).to(dtype), group, perm=perm)
    if fmt == "int8g":
        s = (torch.rand(K // group, N, generator=g) * 0.01 + 1e-3).to(dtype).to(DEV)
        q = torch.randint(-128, 128, (K, N), generator=g, dtype=torch.int8).to(DEV)
        return ops.pack_w8g(q, s, (0.1 * s).to(dtype), group, perm=perm)
    if fmt == "int8":
        q = torch.randint(-128, 128, (K, N), generator=g, dtype=torch.int8).to(DEV)
        return ops.pack_w8(q, (torch.rand(N, generator=g) * 0.01 + 1e-3).to(dtype).to(DEV))
    return ops.pack_f16(_randn(g, K, N, dtype=dtype, scale=0.03))


def _gemm(fmt, dtype=F16, B=1, K=1024, N=512, group=128, bias=False, silu=False, act_order=False):
    from rtp_llm_b200 import ops

    def setup():
        g = _gen(99)
        perm = torch.randperm(K, generator=g) if act_order else None
        w = _weight(fmt, dtype, K, N, g, group, perm)
        static = dict(w=w)
        if bias:
            static["bias"] = _randn(g, N, dtype=dtype)
        outs = {"y": ((B, N // 2 if silu else N), dtype)}
        if act_order:
            outs["x_perm"] = ((B, K), dtype)

        def call(b):
            ops.wo_gemm(b["x"], b["w"], b["ws"], bias=b.get("bias"), out=b["y"], silu_mul=silu, x_perm=b.get("x_perm"))
        ws = ops.gemm_workspace(B, [(K, N)], DEV).numel()
        return Spec(lambda seed: dict(x=_randn(_gen(seed), B, K, dtype=dtype)), call, static, outs=outs,
                    ws={"ws": (ws, 16384 + 2048 * 4)})
    return setup


def _gemm_rs(fmt, dtype=F16, B=5, K=1024, N=1024, world=2, rank=0):
    """b200_wo_gemm_rs of one rank into plain regions on one device (as tests/test_gpu_peer_one_gpu.py runs it): the epilogue
    pushes the other rank's columns into its region and reads the call counter in its own; both regions are in place."""
    import ctypes

    from rtp_llm_b200 import _lib
    max_msg = B * N * 2

    def setup():
        lib = _lib.load()
        nbytes = int(lib.b200_peer_ar_region_bytes(max_msg))
        w = _weight(fmt, dtype, K, N, _gen(77))

        def dyn(seed):
            g = _gen(seed)
            d = dict(x=_randn(g, B, K, dtype=dtype))
            for q in range(world):
                d[f"region{q}"] = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8).to(DEV)
            return d

        def call(b):
            regions = (ctypes.c_void_p * world)(*[b[f"region{q}"].data_ptr() for q in range(world)])
            _lib.check(lib.b200_wo_gemm_rs(w.fmt, int(dtype == BF16), b["x"].data_ptr(), B, K, N, w.data.data_ptr(),
                                           None if w.col_scale is None else w.col_scale.data_ptr(), None, b["y"].data_ptr(), None,
                                           0, 0, regions, max_msg, rank, world, torch.cuda.current_stream().cuda_stream),
                       "b200_wo_gemm_rs")
        return Spec(dyn, call, inplace=tuple(f"region{q}" for q in range(world)), outs={"y": ((B, N), dtype)})
    return setup


GEMM = [
    Case("gemm int4 g128 b1 unsplit", ("wo_gemm_kernel",), _gemm("int4"), {SPLITK: 1}),
    Case("gemm int4 g128 b33 l2 merge bf16 bias", ("wo_gemm_kernel",), _gemm("int4", BF16, B=33, bias=True), {SPLITK: 4}),
    Case("gemm int4 g64 b1 l2 merge", ("wo_gemm_kernel",), _gemm("int4", group=64), {SPLITK: 4}),
    Case("gemm int4 g32 b128 bf16", ("wo_gemm_kernel",), _gemm("int4", BF16, B=128, group=32), {SPLITK: 2}),
    Case("gemm int8 b33 l2 merge", ("wo_gemm_kernel",), _gemm("int8", B=33), {SPLITK: 8}),
    Case("gemm int8g b1 bf16 silu_mul", ("wo_gemm_kernel",), _gemm("int8g", BF16, silu=True), {SPLITK: 2}),
    Case("gemm f16 b128 unsplit bias", ("wo_gemm_kernel",), _gemm("f16", B=128, bias=True), {SPLITK: 1}),
    Case("gemm f16 b1 l2 merge silu_mul", ("wo_gemm_kernel",), _gemm("f16", silu=True), {SPLITK: 4}),
    Case("gemm_rs int4 rank 0 of 2 cluster merge", ("wo_gemm_kernel/rs",), _gemm_rs("int4"), {SPLITK: 2}),
    Case("gemm_rs f16 rank 1 of 2 unsplit bf16", ("wo_gemm_kernel/rs",), _gemm_rs("f16", BF16, rank=1), {SPLITK: 1}),
    Case("gemm act-order int4 permute_cols", ("permute_cols_kernel", "wo_gemm_kernel"), _gemm("int4", B=5, act_order=True),
         {SPLITK: 2}),
]


# ---------------------------------------------------------------------------------------------- glue
def _add_rmsnorm(hidden, rows, residual, dtype=F16):
    from rtp_llm_b200 import ops

    def setup():
        gamma = (1 + 0.3 * torch.randn(hidden, generator=_gen(5))).to(dtype).to(DEV)

        def dyn(seed):
            g = _gen(seed)
            d = dict(x=_randn(g, rows, hidden, dtype=dtype))
            if residual:
                d["res"] = _randn(g, rows, hidden, dtype=dtype)
            return d
        return Spec(dyn, lambda b: ops.add_rmsnorm(b["x"], b.get("res"), b["gamma"], 1e-6, out=b["y"]), dict(gamma=gamma),
                    inplace=("res",) if residual else (), outs={"y": ((rows, hidden), dtype)})
    return setup


def _qk_rmsnorm(dtype=BF16, rows=4, Hq=8, Hkv=2, D=128):
    from rtp_llm_b200 import ops

    def setup():
        g = _gen(6)
        static = dict(qg=_randn(g, D, dtype=dtype), kg=_randn(g, D, dtype=dtype))
        return Spec(lambda s: dict(qkv=_randn(_gen(s), rows, (Hq + 2 * Hkv) * D, dtype=dtype)),
                    lambda b: ops.qk_rmsnorm(b["qkv"], b["qg"], b["kg"], Hq, Hkv, D, 1e-6), static, inplace=("qkv",))
    return setup


def _silu(dtype=F16, rows=9, inter=4096):
    from rtp_llm_b200 import ops

    def setup():
        return Spec(lambda s: dict(gu=_randn(_gen(s), rows, 2 * inter, dtype=dtype, scale=3.0)),
                    lambda b: ops.silu_and_mul(b["gu"], out=b["y"]), outs={"y": ((rows, inter), dtype)})
    return setup


def _rope(kind, dtype=F16, B=3, q_len=1, Hq=8, Hkv=2, D=128, T=16, qk_norm=False):
    """kind "plain": b200_rope_append(_multi) / b200_qk_norm_rope_append; "ex": the _ex entries over half the head, with the
    cos/sin table, position ids and logn."""
    from rtp_llm_b200 import rope as rp
    max_len = 256
    M = max_len // T
    P = B * 2 * M + 1
    spec = rp.RopeSpec(dim=D, base=10000.0) if kind == "plain" else rp.RopeSpec(dim=D // 2, max_pos=512)

    def dyn(seed):
        g = _gen(seed)
        d = dict(qkv=_randn(g, B * q_len, (Hq + 2 * Hkv) * D, dtype=dtype, scale=3.0), pool=_randn(g, P, 2, Hkv, T, D, dtype=dtype),
                 pl=_page_list(g, B, M, P), seq=_ints(g, 0, max_len - q_len, B))
        if kind == "ex":
            d["pid"] = _ints(g, 0, 3000, B * q_len)
        return d

    def setup():
        static = {}
        rp.table(spec, DEV)                                  # uploaded here, not inside the call
        if qk_norm:
            g = _gen(8)
            static = dict(qg=_randn(g, D, dtype=dtype), kg=_randn(g, D, dtype=dtype))

        def call(b):
            rp.rope_append(spec, b["qkv"], b["pool"], b["pl"], b["seq"], Hq, q_out=b["q"], q_len=q_len,
                           use_logn_attn=kind == "ex", position_ids=b.get("pid"),
                           qk_norm=(b["qg"], b["kg"], 1e-6) if qk_norm else None)
        return Spec(dyn, call, static, inplace=("pool",), outs={"q": ((B * q_len, Hq * D), dtype)})
    return setup


def _kv_compact(dtype=BF16, B=3, n=8, Hkv=2, D=128, T=16, layers=2):
    from rtp_llm_b200 import ops
    from tests.verify_oracle import ancestors, random_tree
    max_len = 256
    M = max_len // T
    P = B * 2 * M + 1

    def dyn(seed):
        g = _gen(seed)
        rng = np.random.default_rng(seed)
        path = np.full((B, n), -1, np.int32)
        acc = np.zeros(B, np.int32)
        for b in range(B):
            chain = ancestors(random_tree(rng, n, "random"))[int(rng.integers(1, n))]
            path[b, : len(chain)] = chain
            acc[b] = len(chain) - 1
        d = {f"pool{i}": _randn(g, P, 2, Hkv, T, D, dtype=dtype) for i in range(layers)}
        d.update(pl=_page_list(g, B, M, P), seq=_ints(g, 0, max_len - n, B), path=torch.from_numpy(path).to(DEV),
                 acc=torch.from_numpy(acc).to(DEV))
        return d

    def setup():
        return Spec(dyn, lambda b: ops.kv_compact_path([b[f"pool{i}"] for i in range(layers)], b["pl"], b["seq"], b["path"], b["acc"]),
                    inplace=tuple(f"pool{i}" for i in range(layers)))
    return setup


GLUE = [
    Case("add_rmsnorm residual f16", ("add_rmsnorm_kernel",), _add_rmsnorm(4096, 7, True)),
    Case("add_rmsnorm no residual bf16", ("add_rmsnorm_kernel",), _add_rmsnorm(2048, 33, False, BF16)),
    Case("add_rmsnorm hidden 12288 residual bf16", ("add_rmsnorm_kernel",), _add_rmsnorm(12288, 3, True, BF16)),
    Case("qk_rmsnorm bf16", ("qk_rmsnorm_kernel",), _qk_rmsnorm()),
    Case("silu_and_mul f16", ("silu_and_mul_kernel",), _silu()),
    Case("rope_append f16", ("rope_append_kernel",), _rope("plain")),
    Case("rope_append_multi bf16", ("rope_append_kernel",), _rope("plain", BF16, q_len=4)),
    Case("rope_append_ex f16", ("rope_append_kernel",), _rope("ex")),
    Case("rope_append_ex_multi bf16", ("rope_append_kernel",), _rope("ex", BF16, q_len=3)),
    Case("qk_norm_rope_append bf16", ("rope_append_kernel",), _rope("plain", BF16, q_len=2, qk_norm=True)),
    Case("qk_norm_rope_append_ex f16", ("rope_append_kernel",), _rope("ex", qk_norm=True)),
    Case("kv_compact_path bf16", ("kv_compact_path_kernel",), _kv_compact()),
]


# ---------------------------------------------------------------------------------------------- endings
def _sample(min_p=False, B=4, V=3000, H=16):
    from rtp_llm_b200 import ops

    def dyn(seed):
        g = _gen(seed)
        d = dict(logits=_randn(g, B, V, dtype=F32, scale=3.0), top_k=_ints(g, 0, 60, B),
                 top_p=(0.6 + 0.4 * torch.rand(B, generator=g)).to(DEV), uniform=torch.rand(B, generator=g).to(DEV),
                 temp=(0.5 + torch.rand(B, generator=g)).to(DEV), hist=_ints(g, 0, V, B, H), hist_len=_ints(g, 1, H + 1, B),
                 rep=(1 + 0.5 * torch.rand(B, generator=g)).to(DEV), pres=(0.5 * torch.rand(B, generator=g)).to(DEV),
                 freq=(0.5 * torch.rand(B, generator=g)).to(DEV))
        if min_p:
            d["min_p"] = (0.2 * torch.rand(B, generator=g)).to(DEV)
        return d

    def call(b):
        ops.sample(b["logits"], b["top_k"], b["top_p"], b["uniform"], temperature=b["temp"], history=b["hist"],
                   hist_len=b["hist_len"], repetition=b["rep"], presence=b["pres"], frequency=b["freq"], count_ws=b["count"],
                   out=dict(token=b["token"], token_prob=b["token_prob"], probs=b["probs"]), min_p=b.get("min_p"))

    def setup():
        return Spec(dyn, call, inplace=("logits",), outs=dict(token=((B,), I32), token_prob=((B,), F32), probs=((B, V), F32)),
                    ws=dict(count=(B * V * 4, 0)))
    return setup


def _spec_verify(sampling, B=4, n=4, V=500):
    from rtp_llm_b200 import ops

    def dyn(seed):
        g = _gen(seed)
        if sampling:
            return dict(drafts=_ints(g, 0, V, B, n), tp=torch.softmax(torch.randn(B, n + 1, V, generator=g) * 2, -1).to(DEV),
                        dp=torch.softmax(torch.randn(B, n, V, generator=g) * 2, -1).to(DEV),
                        u=torch.rand(B, n + 1, generator=g).to(DEV))
        tid = torch.randint(0, 8, (B, n + 1), generator=g, dtype=I32)
        drafts = torch.where(torch.rand(B, n, generator=g) < 0.8, tid[:, :n], (tid[:, :n] + 1) % 8)
        return dict(drafts=drafts.to(DEV), tid=tid.to(DEV))

    def call(b):
        if sampling:
            ops.spec_verify(b["drafts"], target_probs=b["tp"], draft_probs=b["dp"], uniform=b["u"], out_tokens=b["tok"],
                            accepted=b["acc"])
        else:
            ops.spec_verify(b["drafts"], target_ids=b["tid"], out_tokens=b["tok"], accepted=b["acc"])

    def setup():
        return Spec(dyn, call, outs=dict(tok=((B, n + 1), I32), acc=((B,), I32)))
    return setup


def _spec_verify_tree(B=4, n=8):
    from rtp_llm_b200 import ops
    from tests.verify_oracle import random_tree

    def dyn(seed):
        g = _gen(seed)
        rng = np.random.default_rng(seed)
        par = torch.from_numpy(np.stack([random_tree(rng, n, "random") for _ in range(B)])).to(I32)
        tok = torch.randint(0, 3, (B, n), generator=g, dtype=I32)
        return dict(par=par.to(DEV), tok=tok.to(DEV), tid=torch.randint(0, 3, (B, n), generator=g, dtype=I32).to(DEV))

    def setup():
        return Spec(dyn, lambda b: ops.spec_verify_tree(b["par"], b["tok"], target_ids=b["tid"], out_tokens=b["o"], accepted=b["a"],
                                                         accepted_path=b["p"]),
                    outs=dict(o=((B, n), I32), a=((B,), I32), p=((B, n), I32)))
    return setup


BEAM_OUT = ("cand_token", "cand_parent", "cand_score", "next_token", "next_parent", "next_cum")


def _beam_step(dtype=F32, B=3, W=4, V=2000, eos=7):
    from rtp_llm_b200 import ops

    def dyn(seed):
        g = _gen(seed)
        logits = torch.randn(B * W, V, generator=g) * 3
        logits[::2, eos] += 6.0
        return dict(logits=logits.to(dtype).to(DEV), cum=(-5 * torch.rand(B, W, generator=g)).to(DEV))

    def setup():
        shapes = dict(cand_token=((B, 2 * W), I32), cand_parent=((B, 2 * W), I32), cand_score=((B, 2 * W), F32),
                      next_token=((B, W), I32), next_parent=((B, W), I32), next_cum=((B, W), F32))
        ws = ops.beam_search_workspace(B, W, V, DEV).numel()
        return Spec(dyn, lambda b: ops.beam_search_step(b["logits"], b["cum"], W, eos, workspace=b["ws"],
                                                        out={k: b[k] for k in BEAM_OUT}),
                    outs=shapes, ws=dict(ws=(ws, 0)))
    return setup


def _beam_hyps(stage, B=3, W=4, max_len=16, H=12, eos=5):
    """stage "update": b200_beam_hypotheses_update on a state that already holds hypotheses; "finalize": its finalize."""
    from rtp_llm_b200 import ops

    def candidates(g):
        score, _ = torch.sort(-10 * torch.rand(B, 2 * W, generator=g), dim=1, descending=True)
        return dict(cand_token=torch.randint(0, 8, (B, 2 * W), generator=g, dtype=I32).to(DEV),
                    cand_parent=torch.randint(0, W, (B, 2 * W), generator=g, dtype=I32).to(DEV), cand_score=score.to(DEV))

    def dyn(seed):
        g = _gen(seed)
        d = dict(hist=_ints(g, 0, 8, B * W, H), hist_len=_ints(g, 2, H + 1, B * W), lp=torch.rand(B, generator=g).to(DEV) + 0.5,
                 es=_ints(g, 0, 3, B), state=ops.beam_hypotheses_state(B, W, max_len, DEV), done=torch.zeros(B, dtype=I32, device=DEV))
        ops.beam_hypotheses_update(candidates(g), d["hist"], d["hist_len"], eos, d["lp"], d["es"], d["state"], d["done"], max_len)
        d.update(candidates(g))
        d["cum"] = (-5 * torch.rand(B, W, generator=g)).to(DEV)
        torch.cuda.synchronize()
        return d

    def setup():
        if stage == "update":
            call = (lambda b: ops.beam_hypotheses_update({k: b[k] for k in BEAM_OUT[:3]}, b["hist"], b["hist_len"], eos, b["lp"],
                                                          b["es"], b["state"], b["done"], max_len))
            return Spec(dyn, call, inplace=("state", "done"))
        shapes = dict(tokens=((B, W, max_len), I32), len=((B, W), I32), score=((B, W), F32), cum_out=((B, W), F32))

        def call(b):
            ops.beam_hypotheses_finalize(b["state"], b["done"], b["cum"], b["hist"], b["hist_len"], W, max_len, b["lp"],
                                         out=dict(tokens=b["tokens"], len=b["len"], score=b["score"], cum=b["cum_out"]))
        return Spec(dyn, call, outs=shapes)
    return setup


def _logprobs(dtype=F16, rows=5, V=5000, top_n=8):
    from rtp_llm_b200 import ops

    def setup():
        ws = ops.token_logprobs_workspace(rows, V, top_n, DEV).numel()
        return Spec(lambda s: dict(logits=_randn(_gen(s), rows, V, dtype=dtype, scale=3.0), tok=_ints(_gen(s + 50), 0, V, rows)),
                    lambda b: ops.token_logprobs(b["logits"], top_n, b["tok"], workspace=b["ws"],
                                                 out=dict(token_logprob=b["lp"], top_ids=b["ids"], top_logprobs=b["top"])),
                    outs=dict(lp=((rows,), F32), ids=((rows, top_n), I32), top=((rows, top_n), F32)), ws=dict(ws=(ws, 0)))
    return setup


def _ban_ngram(dtype=BF16, rows=4, V=1000, H=24):
    from rtp_llm_b200 import ops

    def dyn(seed):
        g = _gen(seed)
        return dict(logits=_randn(g, rows, V, dtype=dtype), hist=_ints(g, 0, 4, rows, H), hist_len=_ints(g, 4, H + 1, rows),
                    ngram=_ints(g, 1, 4, rows))

    def setup():
        return Spec(dyn, lambda b: ops.ban_repeat_ngram(b["logits"], b["hist"], b["hist_len"], b["ngram"]), inplace=("logits",))
    return setup


def _constrain(dtype=F32, rows=4, V=3000, per_row=16):
    from rtp_llm_b200 import ops
    words = (V + 31) // 32

    def dyn(seed):
        g = _gen(seed)
        cuts = torch.sort(torch.randint(0, rows * per_row + 1, (rows - 1,), generator=g)).values
        offsets = torch.cat([torch.zeros(1, dtype=torch.int64), cuts, torch.tensor([rows * per_row])]).to(I32)
        ids = torch.cat([torch.randperm(V, generator=g)[: int(offsets[r + 1] - offsets[r])] for r in range(rows)]).to(I32)
        return dict(logits=_randn(g, rows, V, dtype=dtype, scale=3.0),
                    mask=torch.randint(-2 ** 31, 2 ** 31 - 1, (rows, words), generator=g, dtype=I32).to(DEV),
                    off=offsets.to(DEV), ids=ids.to(DEV), val=(4 * torch.randn(rows * per_row, generator=g)).to(DEV))

    def setup():
        return Spec(dyn, lambda b: ops.constrain_logits(b["logits"], b["mask"], (b["off"], b["ids"], b["val"])),
                    inplace=("logits",))
    return setup


ENDINGS = [
    Case("sample penalties history", ("sample_kernel",), _sample()),
    Case("sample penalties min_p", ("sample_kernel",), _sample(min_p=True), stream=False),
    Case("spec_verify greedy", ("spec_verify_kernel",), _spec_verify(False)),
    Case("spec_verify sampling", ("spec_verify_kernel",), _spec_verify(True)),
    Case("spec_verify_tree greedy", ("spec_verify_kernel",), _spec_verify_tree()),
    Case("beam_search_step fp32", ("beam_search_kernel",), _beam_step()),
    Case("beam_search_step f16", ("beam_search_kernel",), _beam_step(F16)),
    Case("beam_hypotheses_update", ("beam_hyps_update_kernel",), _beam_hyps("update")),
    Case("beam_hypotheses_finalize", ("beam_hyps_finalize_kernel",), _beam_hyps("finalize")),
    Case("token_logprobs f16", ("token_logprobs_kernel",), _logprobs()),
    Case("ban_repeat_ngram bf16", ("ban_repeat_ngram_kernel",), _ban_ngram()),
    Case("constrain_logits fp32", ("constrain_logits_kernel",), _constrain()),
    Case("constrain_logits f16", ("constrain_logits_kernel",), _constrain(F16)),
]


# ---------------------------------------------------------------------------------------------- decode program
def _program(fmt, B, dtype=F16, K=1024, Hq=8, Hkv=2, D=128, T=16):
    """One recorded program whose segment holds GEMM -> norm -> rope -> GEMM (decode_segment_kernel), launched with PDL."""
    from rtp_llm_b200 import ops
    N1 = (Hq + 2 * Hkv) * D
    max_len = 256
    M = max_len // T
    P = B * 2 * M + 1

    def dyn(seed):
        g = _gen(seed)
        return dict(x=_randn(g, B, K, dtype=dtype), res=_randn(g, B, N1, dtype=dtype), pool=_randn(g, P, 2, Hkv, T, D, dtype=dtype),
                    pl=_page_list(g, B, M, P), seq=_ints(g, 0, max_len - 1, B))

    def setup():
        g = _gen(42)
        static = dict(w1=_weight(fmt, dtype, K, N1, g), w2=_weight(fmt, dtype, Hq * D, 512, g),
                      gamma=(1 + 0.3 * torch.randn(N1, generator=g)).to(dtype).to(DEV))
        ws = ops.gemm_workspace(B, [(K, N1), (Hq * D, 512)], DEV).numel()
        holder = {}

        def call(b):
            key = tuple(v.data_ptr() for v in b.values() if isinstance(v, torch.Tensor))
            if holder.get("key") != key:
                prog = ops.Program()
                with prog.record():
                    ops.wo_gemm(b["x"], b["w1"], b["ws"], out=b["qkv"])
                    ops.add_rmsnorm(b["qkv"], b["res"], b["gamma"], 1e-6, out=b["qkvn"])
                    ops.rope_append(b["qkvn"], b["pool"], b["pl"], b["seq"], Hq, 10000.0, q_out=b["q"])
                    ops.wo_gemm(b["q"], b["w2"], b["ws"], out=b["y"])
                assert prog.num_launches == 1, f"expected one persistent-kernel launch, got {prog.num_launches}"
                holder.update(key=key, prog=prog)
            holder["prog"].launch()
        outs = dict(qkv=((B, N1), dtype), qkvn=((B, N1), dtype), q=((B, Hq * D), dtype), y=((B, 512), dtype))
        return Spec(dyn, call, static, inplace=("res", "pool"), outs=outs, ws=dict(ws=(ws, 16384 + 2048 * 4)))
    return setup


PROGRAM = [
    Case("program int4 b3", ("decode_segment_kernel",), _program("int4", 3)),
    Case("program int8 b40 bf16", ("decode_segment_kernel",), _program("int8", 40, BF16)),
]

CASES = ATTN + GEMM + GLUE + ENDINGS + PROGRAM
