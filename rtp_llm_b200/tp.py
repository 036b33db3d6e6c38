"""Tensor-parallel collectives of the decode path: SUM all-reduce of [B, hidden] after each row-parallel GEMM
(reference: distributed/collective_torch.py:694-722, call sites hybrid/causal_attention.py:91-92, dense_mlp.py:104-105)
and the all-gather of vocab-split logits (cpp/models/PyWrappedModel.cc:915-936).  One process per GPU,
torch.distributed (NCCL over NVLink 4 / NVSwitch) as plumbing; both calls are CUDA-graph capturable."""
from __future__ import annotations

import torch
import torch.distributed as dist


class NcclComm:
    """Stock NCCL collectives on the TP group (the baseline arm; see PeerComm in this module for the custom kernel)."""

    def __init__(self, device: torch.device, group=None):
        self.device, self.group = device, group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)

    def all_reduce(self, t: torch.Tensor) -> None:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)

    def all_gather(self, out: torch.Tensor, t: torch.Tensor) -> None:
        dist.all_gather_into_tensor(out, t, group=self.group)


class PeerComm(NcclComm):
    """TP all-reduce through our own one-shot kernel over NVLink peer memory (csrc/peer_allreduce.cuh): each rank
    cudaMalloc's a peer-visible region, the 64-byte IPC handles travel over the existing process group, and the kernel
    reads all peers' slots directly. The (once per step, 2 MB) logits all-gather stays on NCCL."""

    MAX_MESSAGE = 1 << 19   # decode all-reduces are [B, hidden] fp16: 256 KiB at the BASELINE configs (region = 16 MiB)

    def __init__(self, device: torch.device, group=None):
        super().__init__(device, group)
        import ctypes
        from . import _lib
        lib = _lib.load()
        self._lib, self._ct = lib, ctypes
        nbytes = lib.b200_peer_ar_region_bytes(self.MAX_MESSAGE)
        mine = ctypes.c_void_p()
        handle = ctypes.create_string_buffer(64)
        _lib.check(lib.b200_peer_alloc(nbytes, ctypes.byref(mine), handle), "b200_peer_alloc")
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle.raw), group=group)
        ptrs = []
        for r in range(self.world):
            if r == self.rank:
                ptrs.append(mine.value)
            else:
                p = ctypes.c_void_p()
                hb = ctypes.create_string_buffer(handles[r], 64)
                _lib.check(lib.b200_peer_open(hb, ctypes.byref(p)), "b200_peer_open")
                ptrs.append(p.value)
        self._regions = (ctypes.c_void_p * self.world)(*ptrs)
        dist.barrier(group=group)     # every rank has zeroed + mapped every region before the first kernel

    def all_reduce(self, t: torch.Tensor) -> None:
        from . import _lib
        nbytes = t.numel() * t.element_size()
        if nbytes > self.MAX_MESSAGE or nbytes % 16 or not t.is_contiguous():
            return super().all_reduce(t)
        _lib.check(self._lib.b200_peer_allreduce(t.data_ptr(), t.data_ptr(), nbytes, 1 if t.dtype == torch.bfloat16 else 0,
                                                 self._regions, self.MAX_MESSAGE, 0, self.rank, self.world,
                                                 torch.cuda.current_stream().cuda_stream), "b200_peer_allreduce")

    def all_reduce_norm(self, t: torch.Tensor, residual: torch.Tensor, gamma: torch.Tensor, eps: float, out: torch.Tensor) -> bool:
        """out = rmsnorm(allreduce(t) + residual) * gamma, residual += allreduce(t), in one kernel. Returns False (nothing
        done) when the shape is outside what the fused kernel covers: the caller then issues the two ops separately."""
        from . import _lib
        rows, hidden = t.shape
        if (rows * hidden * t.element_size() > self.MAX_MESSAGE or hidden % (8 * self.world) or hidden > 8192
                or not (t.is_contiguous() and residual.is_contiguous() and out.is_contiguous())):
            return False
        _lib.check(self._lib.b200_peer_allreduce_norm(t.data_ptr(), residual.data_ptr(), gamma.data_ptr(), out.data_ptr(),
                                                      1 if t.dtype == torch.bfloat16 else 0, rows, hidden, eps, self._regions,
                                                      self.MAX_MESSAGE, self.rank, self.world,
                                                      torch.cuda.current_stream().cuda_stream), "b200_peer_allreduce_norm")
        return True

    def gemm_rs_supported(self, rows: int, hidden: int, elem_size: int = 2) -> bool:
        return (rows * hidden * elem_size <= self.MAX_MESSAGE and hidden % (8 * self.world) == 0 and hidden % 128 == 0
                and hidden <= 8192 and rows <= 128)

    def gemm_rs(self, x: torch.Tensor, w, workspace: torch.Tensor, out: torch.Tensor, pdl: bool = False, bias=None) -> None:
        """Row-parallel GEMM whose epilogue pushes the reduce-scatter words to their owners (b200_wo_gemm_rs); must be
        followed by gather_norm() on `out`."""
        from . import _lib
        B, K = x.shape
        _lib.check(self._lib.b200_wo_gemm_rs(w.fmt, 1 if x.dtype == torch.bfloat16 else 0, x.data_ptr(), B, K, w.N, w.data.data_ptr(),
                                             w.col_scale.data_ptr() if w.col_scale is not None else None,
                                             bias.data_ptr() if bias is not None else None, out.data_ptr(), workspace.data_ptr(),
                                             workspace.numel(), _lib.B200_GEMM_PDL if pdl else 0, self._regions, self.MAX_MESSAGE,
                                             self.rank, self.world, torch.cuda.current_stream().cuda_stream), "b200_wo_gemm_rs")

    def gather_norm(self, t: torch.Tensor, residual: torch.Tensor, gamma: torch.Tensor, eps: float, out: torch.Tensor) -> None:
        """Second half of gemm_rs(): reduce own slice + all-gather + residual add + RMSNorm (b200_peer_gather_norm)."""
        from . import _lib
        rows, hidden = t.shape
        _lib.check(self._lib.b200_peer_gather_norm(t.data_ptr(), residual.data_ptr(), gamma.data_ptr(), out.data_ptr(),
                                                   1 if t.dtype == torch.bfloat16 else 0, rows, hidden, eps, self._regions,
                                                   self.MAX_MESSAGE, self.rank, self.world,
                                                   torch.cuda.current_stream().cuda_stream), "b200_peer_gather_norm")

    def argmax(self, logits: torch.Tensor, vocab_total: int, out: torch.Tensor) -> None:
        """Greedy token over the vocab-split logits (rank r holds columns [r*V_local, (r+1)*V_local))."""
        from . import _lib
        rows, vloc = logits.shape
        _lib.check(self._lib.b200_peer_argmax(logits.data_ptr(), 1 if logits.dtype == torch.bfloat16 else 0, rows, vloc,
                                              vocab_total, out.data_ptr(), self._regions, self.MAX_MESSAGE, self.rank, self.world,
                                              torch.cuda.current_stream().cuda_stream), "b200_peer_argmax")


def make_comm(device: torch.device, group=None, kind: str = "peer"):
    """kind: "peer" (our NVLink kernel) or "nccl" (stock collectives, the baseline arm)."""
    return PeerComm(device, group) if kind == "peer" else NcclComm(device, group)


# ------------------------------------------------------------------------------------------------ sharding
# The reference's tensor-parallel split (rtp_llm/utils/model_weight.py:1489-1580): qkv column-parallel BY HEAD (sp_head,
# :472-491), o row-parallel (sp_0), w1/w3 column-parallel (ffn_sp_neg1_w13, :997), w2 row-parallel (ffn_sp_0, :238),
# scales / zeros split alongside, lm_head vocab rows (sp_0_pad8, :1491). Weights are the loader's UN-permuted tuples
# (fmt, w, scales, zeros_x_scales): int4 w = uint8 [K, N/2]; int8 w = int8 [K, N], scales [N]; int8g w = int8 [K, N], scales /
# zeros_x_scales [K/g, N]; f16 w = [K, N].

def _cols(wt, col_ranges):
    """Select logical output columns [a, b) ranges of a reference-layout weight tuple."""
    fmt, w, s, zs = wt
    if fmt == "int4":
        assert all(a % 2 == 0 and b % 2 == 0 for a, b in col_ranges)
        wq = torch.cat([w[:, a // 2:b // 2] for a, b in col_ranges], dim=1).contiguous()
        return (fmt, wq, torch.cat([s[:, a:b] for a, b in col_ranges], 1).contiguous(),
                torch.cat([zs[:, a:b] for a, b in col_ranges], 1).contiguous())
    wq = torch.cat([w[:, a:b] for a, b in col_ranges], dim=1).contiguous()
    if fmt == "int8g":
        return (fmt, wq, torch.cat([s[:, a:b] for a, b in col_ranges], 1).contiguous(),
                torch.cat([zs[:, a:b] for a, b in col_ranges], 1).contiguous())
    if fmt == "int8":
        return (fmt, wq, torch.cat([s[a:b] for a, b in col_ranges]).contiguous(), None)
    return (fmt, wq, None, None)


def _rows(wt, a, b, group=128):
    """Select input rows (the contraction dim) [a, b); group-wise scales follow in units of `group`."""
    fmt, w, s, zs = wt
    if fmt in ("int4", "int8g"):
        assert a % group == 0 and b % group == 0, "row-parallel group-wise shards must align to the quantisation group"
        return (fmt, w[a:b].contiguous(), s[a // group:b // group].contiguous(), zs[a // group:b // group].contiguous())
    return (fmt, w[a:b].contiguous(), s, None)


def shard_qkv(wt, head_num, kv_head_num, head_dim, rank, tp):
    hq, hkv = head_num // tp, max(kv_head_num // tp, 1)
    kv_rank = rank if kv_head_num >= tp else rank * kv_head_num // tp      # replicated kv heads when Hkv < tp
    q0 = rank * hq * head_dim
    k_base, v_base = head_num * head_dim, (head_num + kv_head_num) * head_dim
    k0 = k_base + kv_rank * hkv * head_dim
    v0 = v_base + kv_rank * hkv * head_dim
    return _cols(wt, [(q0, q0 + hq * head_dim), (k0, k0 + hkv * head_dim), (v0, v0 + hkv * head_dim)])


def shard_o(wt, head_num, head_dim, rank, tp):
    k = head_num // tp * head_dim
    return _rows(wt, rank * k, (rank + 1) * k)


def shard_w13(wt, inter, rank, tp):
    i = inter // tp
    return _cols(wt, [(rank * i, (rank + 1) * i), (inter + rank * i, inter + (rank + 1) * i)])


def shard_w2(wt, inter, rank, tp):
    i = inter // tp
    return _rows(wt, rank * i, (rank + 1) * i)


def shard_lm_head(wt, vocab_local, rank):
    fmt, w, s, zs = wt
    a, b = rank * vocab_local, (rank + 1) * vocab_local
    part = w[:, a:min(b, w.shape[1])]
    if part.shape[1] < vocab_local:                                          # sp_0_pad8: pad the last shard with zeros
        part = torch.cat([part, torch.zeros(w.shape[0], vocab_local - part.shape[1], dtype=w.dtype, device=w.device)], 1)
    return (fmt, part.contiguous(), None, None)
