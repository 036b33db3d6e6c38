"""Torch-tensor face of the C ABI. PyTorch is plumbing here (device memory + streams); all compute is in
libb200_decode.so. Every function launches on the current CUDA stream and is CUDA-graph capturable."""
from __future__ import annotations

import math
import numbers
from typing import Mapping, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import (B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT4_G32, B200_FMT_INT4_G64, B200_FMT_INT8, B200_FMT_INT8G, B200Error,
                   check)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _is_bf16(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return 1
    if t.dtype == torch.float16:
        return 0
    raise B200Error(f"unsupported activation dtype {t.dtype} (fp16 / bf16 only)")


def _cuda_contig(*ts: Optional[torch.Tensor]) -> None:
    for t in ts:
        if t is not None and not (t.is_cuda and t.is_contiguous()):
            raise B200Error("expected contiguous CUDA tensors")


def check_lengths(who: str, lengths: torch.Tensor, seqs: int) -> None:
    """Raise unless `lengths` is what a kernel can read through its pointer: int32, contiguous, at least `seqs` entries, in
    device memory or in pinned host memory (which the GPU reads in place). A pageable host tensor would hand the kernel a host
    pointer, and an int64 one would be read as pairs of int32."""
    if not (torch.is_tensor(lengths) and lengths.dtype == torch.int32 and lengths.is_contiguous() and lengths.numel() >= seqs
            and (lengths.is_cuda or lengths.is_pinned())):
        got = (f"{lengths.dtype} [{lengths.numel()}] on {lengths.device}{'' if lengths.is_cuda or lengths.is_pinned() else ', pageable'}"
               if torch.is_tensor(lengths) else type(lengths).__name__)
        raise B200Error(f"{who}: sequence_lengths must be a contiguous int32 tensor of at least {seqs} entries in CUDA or pinned "
                        f"host memory (got {got})")


_DTYPE_NAMES = {torch.int32: "int32", torch.float32: "fp32"}


def _need(who: str, name: str, t: torch.Tensor, dtype: torch.dtype, shape: tuple, flat: bool = False) -> None:
    """Raise "{who}: {name} must be {dtype} [shape]" unless t has that dtype and shape. An int in `shape` is a size, a str a
    free dimension (printed as it is). flat: any shape with the element count of `shape` will do."""
    if flat:
        ok = t.numel() == math.prod(shape)
    else:
        ok = t.dim() == len(shape) and all(isinstance(s, str) or n == s for n, s in zip(t.shape, shape))
    if t.dtype != dtype or not ok:
        raise B200Error(f"{who}: {name} must be {_DTYPE_NAMES[dtype]} [{', '.join(map(str, shape))}]")


def _outputs(who: str, out: Optional[dict], device, **specs) -> dict:
    """`out` (None, or a dict of output tensors; a None entry counts as missing) with each output of specs, name=(dtype,
    shape), that it lacks allocated on `device`. A supplied one must have the dtype and the element count of its spec."""
    out = {k: v for k, v in (out or {}).items() if v is not None}
    for k, (dtype, shape) in specs.items():
        if k not in out:
            out[k] = torch.empty(shape, dtype=dtype, device=device)
        elif out[k].dtype != dtype or out[k].numel() != math.prod(shape):
            raise B200Error(f"{who}: {k} must be {dtype} {list(shape)}")
    return out


def device_check(device: int = 0) -> None:
    check(_lib.load().b200_device_check(device), "b200_device_check")


def set_pdl(enable: bool) -> None:
    """Programmatic dependent launch for the whole decode chain (see include/b200_decode_ops.h)."""
    check(_lib.load().b200_set_pdl(1 if enable else 0), "b200_set_pdl")


def launch_count() -> int:
    return int(_lib.load().b200_launch_count())


# ------------------------------------------------------------------------------------------------ indexing
def convert_block_table(block_ids: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[B,M] int32 -> [B,1,2,M] int32 page list (XQAAttnOp::prepare, XQAAttnOp.cc:77-92)."""
    _cuda_contig(block_ids, out)
    B, M = block_ids.shape
    if out is None:
        out = torch.empty((B, 1, 2, M), dtype=torch.int32, device=block_ids.device)
    check(_lib.load().b200_convert_block_table(_p(out), _p(block_ids), B, M, _stream()), "b200_convert_block_table")
    return out


def paged_attn_plan(sequence_lengths: torch.Tensor, block_ids: Optional[torch.Tensor], tokens_per_block: int,
                    input_lengths: Optional[torch.Tensor] = None, prefix_lengths: Optional[torch.Tensor] = None):
    ref = sequence_lengths if prefix_lengths is None else prefix_lengths
    B = ref.shape[0]
    dev = ref.device
    M = block_ids.shape[1] if block_ids is not None else 0
    ntok = B if prefix_lengths is None else int(input_lengths.sum().item())
    last = torch.zeros(B, dtype=torch.int32, device=dev)
    indptr = torch.zeros(B + 1, dtype=torch.int32, device=dev)
    indice = torch.zeros(max(B * M, 1), dtype=torch.int32, device=dev)
    bidx = torch.zeros(max(ntok, 1), dtype=torch.int32, device=dev)
    pos = torch.zeros(max(ntok, 1), dtype=torch.int32, device=dev)
    check(_lib.load().b200_paged_attn_plan(_p(input_lengths), _p(sequence_lengths), _p(prefix_lengths), _p(block_ids), B,
                                           M, tokens_per_block, _p(last), _p(indptr), _p(indice), _p(bidx), _p(pos),
                                           _stream()), "b200_paged_attn_plan")
    return dict(last_page_len=last, page_indptr=indptr, page_indice=indice, batch_indice=bidx[:ntok], positions=pos[:ntok])


# ------------------------------------------------------------------------------------------------ attention
def attn_workspace(batch: int, head_num: int, kv_head_num: int, max_seq_len: int, device) -> torch.Tensor:
    n = _lib.load().b200_paged_decode_attn_workspace_bytes(batch, head_num, kv_head_num, max_seq_len)
    return torch.zeros(max(int(n), 256), dtype=torch.uint8, device=device)


def _paged_attn(entry: str, q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                max_seq_len: int, workspace: torch.Tensor, out: Optional[torch.Tensor], rows: tuple, seqs: int, Hq: Optional[int],
                extra: tuple, sizes: Optional[tuple] = None) -> torch.Tensor:
    """The call of b200_<entry> that the paged_decode_attn* wrappers share. rows: the sizes before the heads, (B,) or (B, q_len
    or W), passed after head_dim unless `sizes` is passed there instead; seqs: the sequences whose lengths the kernel reads;
    out [*rows, Hq*D] of q's dtype is allocated when not given; Hq None: q's elements over rows * D. extra: the arguments
    between sequence_lengths and the workspace (q_scale among them). Tensors among sizes and extra are checked and passed as
    pointers."""
    sizes = rows if sizes is None else sizes
    _cuda_contig(q, kv_cache_base, page_list, *(t for t in sizes + extra if isinstance(t, torch.Tensor)), workspace, out)
    check_lengths(entry, sequence_lengths, seqs)
    P, two, Hkv, T, D = kv_cache_base.shape
    if Hq is None:
        Hq = q.numel() // (math.prod(rows) * D)
    if out is None:
        out = torch.empty((*rows, Hq * D), dtype=q.dtype, device=q.device)
    arg = lambda a: _p(a) if isinstance(a, torch.Tensor) else a   # tensors go to C as pointers
    check(getattr(_lib.load(), "b200_" + entry)(
        _p(q), _is_bf16(q), _p(out), Hq, Hkv, D, *map(arg, sizes), page_list.shape[-1], max_seq_len, T, _p(kv_cache_base),
        _p(page_list), _p(sequence_lengths), *map(arg, extra), _p(workspace), workspace.numel(), _stream()), "b200_" + entry)
    return out


def paged_decode_attn(q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor,
                      sequence_lengths: torch.Tensor, max_seq_len: int, workspace: torch.Tensor,
                      out: Optional[torch.Tensor] = None, q_scale: float = 1.0) -> torch.Tensor:
    """q [B,Hq,D] (or [B,Hq*D]); kv_cache_base [P,2,Hkv,T,D]; page_list [B,1,2,M]; sequence_lengths [B] int32 = tokens
    already cached; max_seq_len = host bound on sequence_lengths+1. Returns [B, Hq*D]."""
    return _paged_attn("paged_decode_attn", q, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out, (q.shape[0],),
                       q.shape[0], None, (q_scale,))


def paged_decode_attn_multi(q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                            max_seq_len: int, workspace: torch.Tensor, out: Optional[torch.Tensor] = None, q_scale: float = 1.0) -> torch.Tensor:
    """q [B, q_len, Hq, D] (q_len speculative tokens per sequence, K/V already appended); sequence_lengths [B] = tokens cached
    before them; query j attends to positions 0 .. sequence_lengths[b] + j. Returns [B, q_len, Hq*D]."""
    return _paged_attn("paged_decode_attn_multi", q, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out,
                       tuple(q.shape[:2]), q.shape[0], q.shape[2], (q_scale,))


def paged_decode_attn_beam(q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                           shared_lengths: torch.Tensor, max_seq_len: int, workspace: torch.Tensor, out: Optional[torch.Tensor] = None,
                           q_scale: float = 1.0) -> torch.Tensor:
    """q [B, W, Hq, D]: beam i of request b is sequence b * W + i of page_list [B*W, 1, 2, M] and sequence_lengths [B*W];
    shared_lengths [B] int32 = tokens of each request that all its W beams share (their page_list rows are equal over those
    pages), read once for the W beams. The bits of paged_decode_attn on the B * W rows. Returns [B, W, Hq*D]."""
    return _paged_attn("paged_decode_attn_beam", q, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out,
                       tuple(q.shape[:2]), q.shape[0] * q.shape[1], q.shape[2], (shared_lengths, q_scale))


def paged_decode_attn_prefix(q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                             chunk_offsets: torch.Tensor, chunk_rows: torch.Tensor, shared_lengths: torch.Tensor, max_members: int,
                             max_seq_len: int, workspace: torch.Tensor, out: Optional[torch.Tensor] = None,
                             q_scale: float = 1.0) -> torch.Tensor:
    """paged_decode_attn on q [B, Hq, D] with the rows grouped into chunks that read their shared leading pages once: chunk c is
    the rows chunk_rows[chunk_offsets[c] : chunk_offsets[c + 1]] (int32 [chunks + 1] and [B], at most max_members rows each),
    whose page_list rows are equal over the first shared_lengths[c] / T pages (int32 [chunks]). prefix_chunks builds the three
    from a block table. Rows in no chunk are not written. Returns [B, Hq*D]."""
    who = "paged_decode_attn_prefix"
    B, C, D = q.shape[0], shared_lengths.numel(), kv_cache_base.shape[-1]
    _need(who, "chunk_offsets", chunk_offsets, torch.int32, (C + 1,), flat=True)
    _need(who, "chunk_rows", chunk_rows, torch.int32, (B,), flat=True)
    _need(who, "shared_lengths", shared_lengths, torch.int32, ("chunks",))
    out = _outputs(who, {"attn_out": out}, q.device, attn_out=(q.dtype, (B, q.numel() // (B * D) * D)))["attn_out"]
    return _paged_attn(who, q, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out, (B,), B, None, (q_scale,),
                       (B, C, max_members, chunk_offsets, chunk_rows, shared_lengths))


def prefix_chunks(block_ids: torch.Tensor, sequence_lengths: torch.Tensor, tokens_per_block: int,
                  group: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, int]:
    """The chunking of paged_decode_attn_prefix for a batch, from host int32 tensors block_ids [B, M] and sequence_lengths [B]
    (tokens cached) and the GQA group (head_num / kv_head_num). Rows whose block-table rows start with the same block are
    candidates; only blocks a row has wholly cached count (the token a step appends never lands in a shared block). Among them,
    the rows that agree with the first row on at least k whole blocks form a group sharing k * tokens_per_block tokens, k picked
    to maximise the blocks read once fewer ((rows - 1) * k); the rest are grouped again the same way. A row that shares no whole
    block with another becomes a chunk of one sharing 0 tokens, as does a row left alone after groups are cut, in row order,
    into chunks of at most 64 // group rows. Returns (chunk_offsets [chunks + 1], chunk_rows [B], shared_lengths [chunks],
    max_members), int32 host tensors and an int. Meant to run once per batch composition, not per step."""
    if block_ids.dtype != torch.int32 or block_ids.dim() != 2 or block_ids.is_cuda:
        raise B200Error("prefix_chunks: block_ids must be a host int32 [B, M] tensor")
    B, M = block_ids.shape
    _need("prefix_chunks", "sequence_lengths", sequence_lengths, torch.int32, (B,), flat=True)
    if sequence_lengths.is_cuda or B == 0 or tokens_per_block < 1 or not 1 <= group <= 64:
        raise B200Error(f"prefix_chunks: need host tensors, B >= 1, tokens_per_block >= 1 and group in 1..64 (got B {B}, "
                        f"tokens_per_block {tokens_per_block}, group {group})")
    ids = block_ids.tolist()
    whole = [min(int(n) // tokens_per_block, M) for n in sequence_lengths.reshape(-1).tolist()]
    candidates = {}
    for r in range(B):
        candidates.setdefault(ids[r][0] if M else -1 - r, []).append(r)
    groups = []                                   # (rows, shared blocks)
    for members in candidates.values():
        first = ids[members[0]]
        common = {members[0]: whole[members[0]]}  # whole blocks each member shares with the first
        for r in members[1:]:
            n = min(whole[r], whole[members[0]])
            common[r] = next((j for j in range(n) if ids[r][j] != first[j]), n)
        rest = members
        while len(rest) > 1:
            k = max(set(common[r] for r in rest), key=lambda k: (sum(common[r] >= k for r in rest) - 1) * k)
            sub = [r for r in rest if common[r] >= k]
            if k == 0 or len(sub) < 2:
                break
            groups.append((sub, k))
            rest = [r for r in rest if common[r] < k]
        groups += [([r], 0) for r in rest]
    cap = 64 // group
    offsets, rows, shared = [0], [], []
    for members, k in groups:
        for c in range(0, len(members), cap):
            chunk = members[c:c + cap]
            rows += chunk
            offsets.append(len(rows))
            shared.append(k * tokens_per_block if len(chunk) > 1 else 0)
    max_members = max(b - a for a, b in zip(offsets, offsets[1:]))
    i32 = dict(dtype=torch.int32)
    return torch.tensor(offsets, **i32), torch.tensor(rows, **i32), torch.tensor(shared, **i32), max_members


def paged_decode_attn_tree(q: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                           tree_parents: torch.Tensor, max_seq_len: int, workspace: torch.Tensor, out: Optional[torch.Tensor] = None,
                           q_scale: float = 1.0) -> torch.Tensor:
    """q [B, n, Hq, D]: the n nodes of each sequence's speculative token tree (K/V already appended at slots
    sequence_lengths[b] + j); tree_parents int32 [B, n] (node 0 the root, node j under parents[j] in [0, j)). Query j attends to
    the cached positions and to the slots of its ancestors and itself. A chain gives the bits of paged_decode_attn_multi.
    Returns [B, n, Hq*D]."""
    _need("paged_decode_attn_tree", "tree_parents", tree_parents, torch.int32, tuple(q.shape[:2]))
    return _paged_attn("paged_decode_attn_tree", q, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out,
                       tuple(q.shape[:2]), q.shape[0], q.shape[2], (tree_parents, q_scale))


def paged_decode_attn_rope(qkv: torch.Tensor, kv_cache_base: torch.Tensor, page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                           head_num: int, max_seq_len: int, rope_base: float, workspace: torch.Tensor,
                           out: Optional[torch.Tensor] = None, q_scale: float = 1.0) -> torch.Tensor:
    """RoPE + K/V append + paged decode attention in ONE launch: qkv [B, (Hq+2Hkv)*D] un-rotated (the qkv GEMM output);
    kv_cache_base receives the new token's K (rotated) and V. Bit-identical to rope_append() followed by paged_decode_attn()."""
    return _paged_attn("paged_decode_attn_rope", qkv, kv_cache_base, page_list, sequence_lengths, max_seq_len, workspace, out,
                       (qkv.shape[0],), qkv.shape[0], head_num, (q_scale, rope_base))


# ------------------------------------------------------------------------------------------------ weight-only GEMM
_TRAILER_BYTES = 256
_TRAILER_MAGIC = 0x42323030574F4731        # "B200WOG1": [blob | trailer]
_TRAILER_MAGIC_PERM = 0x42323030574F4732   # "B200WOG2": [blob | perm int32 [K] | trailer]


class PackedWeight:
    """A weight in the layout b200_wo_gemm consumes (+ what the epilogue needs).

    Quantised blobs are SELF-DESCRIBING: the uint8 tensor is [blob bytes | 256-byte trailer] with a magic number, the format and
    (K, N, group). The reference loader hands kernels around as plain tensors and copies them freely
    (device_impl.py:296-298 `.contiguous().to(device)`, state-dict round trips): a Python attribute on the tensor would be
    lost there, the trailer travels with the bytes. PackedWeight.from_tensor() rebuilds the description from any copy.

    A GPTQ act-order weight (rows sorted by g_idx, see device.act_order_perm) also carries its row order: the tensor is then
    [blob | perm int32 [K] | trailer] under its own magic, and `perm` is an int32 view into it. Sorted row j is the
    checkpoint's row perm[j], so the GEMM must consume x[:, perm] (wo_gemm gathers it)."""

    def __init__(self, fmt: int, K: int, N: int, data: torch.Tensor, col_scale: Optional[torch.Tensor] = None,
                 perm: Optional[torch.Tensor] = None):
        self.fmt, self.K, self.N, self.data, self.col_scale, self.perm = fmt, K, N, data, col_scale, perm

    @staticmethod
    def _write_trailer(data: torch.Tensor, fmt: int, K: int, N: int, group: int, magic: int = _TRAILER_MAGIC) -> None:
        t = torch.tensor([magic, fmt, K, N, group], dtype=torch.int64)
        data[-_TRAILER_BYTES:-_TRAILER_BYTES + 40] = t.view(torch.uint8).to(data.device)

    @staticmethod
    def from_tensor(data: torch.Tensor, col_scale: Optional[torch.Tensor] = None) -> "PackedWeight":
        if data.dtype != torch.uint8 or data.dim() != 1 or data.numel() <= _TRAILER_BYTES:
            raise B200Error("not a b200 weight blob (expected a 1-D uint8 tensor with a trailer)")
        t = data[-_TRAILER_BYTES:-_TRAILER_BYTES + 40].cpu().view(torch.int64).tolist()
        if t[0] not in (_TRAILER_MAGIC, _TRAILER_MAGIC_PERM):
            raise B200Error("not a b200 weight blob (bad magic): quantised weights must be loaded through B200Impl")
        fmt, K, N = int(t[1]), int(t[2]), int(t[3])
        n = int(_lib.load().b200_wo_gemm_packed_bytes(fmt, K, N))
        perm_bytes = 4 * K if t[0] == _TRAILER_MAGIC_PERM else 0
        if n + perm_bytes + _TRAILER_BYTES != data.numel():
            raise B200Error(f"b200 weight blob has {data.numel()} bytes, expected {n + perm_bytes + _TRAILER_BYTES} for K={K} N={N}")
        data = data if data.is_contiguous() else data.contiguous()
        perm = data[n:n + perm_bytes].view(torch.int32) if perm_bytes else None
        return PackedWeight(fmt, K, N, data, col_scale, perm)


def _blob(n: int, K: int, perm: Optional[torch.Tensor], device) -> torch.Tensor:
    """[n blob bytes (for the pack kernel to fill) | (perm) | zeroed trailer] tensor, so that equal weights give equal bytes;
    with a perm, its int32 bytes are written in place after a host check that it is a permutation of 0..K-1 (the gather
    kernel indexes shared memory with it unchecked)."""
    extra = 0 if perm is None else 4 * K
    blob = torch.empty(n + extra + _TRAILER_BYTES, dtype=torch.uint8, device=device)
    blob[-_TRAILER_BYTES:].zero_()
    if perm is None:
        return blob
    p = perm.detach().to("cpu", torch.int64).reshape(-1)
    if p.numel() != K or not torch.equal(torch.sort(p).values, torch.arange(K)):
        raise B200Error(f"perm must be a permutation of 0..{K - 1} (got {p.numel()} entries)")
    blob[n:n + 4 * K] = p.to(torch.int32).view(torch.uint8).to(device)
    return blob


def _packed(fmt: int, K: int, N: int, blob: torch.Tensor, group: int, n: int, has_perm: bool,
            col_scale: Optional[torch.Tensor] = None) -> PackedWeight:
    PackedWeight._write_trailer(blob, fmt, K, N, group, _TRAILER_MAGIC_PERM if has_perm else _TRAILER_MAGIC)
    return PackedWeight(fmt, K, N, blob, col_scale, blob[n:n + 4 * K].view(torch.int32) if has_perm else None)


_W4_FORMATS = {128: B200_FMT_INT4, 64: B200_FMT_INT4_G64, 32: B200_FMT_INT4_G32}


def w4_format(K: int, group: int, scales: torch.Tensor, zeros_x_scales: torch.Tensor):
    """(blob format, kernel group, scales, zeros_x_scales) for INT4 weights of quantisation group `group` over K rows.

    128, 64 and 32 have their own blob formats (B200_FMT_INT4, _INT4_G64, _INT4_G32). A larger multiple of 128, per-channel
    (group = K, or -1) included, becomes group 128 with each scale / zero*scale row repeated: every weight keeps its own s and
    zero*s, so the dequantised weights are the same bits. Any other group is left for the library to reject."""
    if group == -1:
        group = K
    if group != 128 and (group <= 0 or scales.shape[0] * group != K or zeros_x_scales.shape[0] != scales.shape[0]):
        raise B200Error(f"pack_w4: group {group} does not match K={K} and scales / zeros_x_scales of {scales.shape[0]} / "
                        f"{zeros_x_scales.shape[0]} rows")
    if group > 128 and group % 128 == 0:
        r = group // 128
        return (B200_FMT_INT4, 128, scales.repeat_interleave(r, dim=0).contiguous(),
                zeros_x_scales.repeat_interleave(r, dim=0).contiguous())
    return _W4_FORMATS.get(group, B200_FMT_INT4), group, scales, zeros_x_scales


def pack_w4(q_packed: torch.Tensor, scales: torch.Tensor, zeros_x_scales: torch.Tensor, group: int = 128,
            perm: Optional[torch.Tensor] = None) -> PackedWeight:
    """q_packed uint8/int8 [K,N/2], scales / zeros_x_scales [K/g,N] in the activation dtype (CUDA). The group picks the blob
    format (w4_format); the trailer records the group as given (per-channel: K). perm: the row order of an act-order weight
    whose rows were sorted by g_idx (PackedWeight), stored in the blob."""
    _cuda_contig(q_packed, scales, zeros_x_scales)
    K, N = q_packed.shape[0], q_packed.shape[1] * 2
    fmt, kernel_group, scales, zeros_x_scales = w4_format(K, group, scales, zeros_x_scales)
    n = _lib.load().b200_wo_gemm_packed_bytes(fmt, K, N)
    if n == 0:
        raise B200Error(f"pack_w4: unsupported shape K={K} N={N}")
    blob = _blob(int(n), K, perm, q_packed.device)
    check(_lib.load().b200_pack_w4(_p(q_packed), _p(scales), _p(zeros_x_scales), K, N, kernel_group, _p(blob), _stream()),
          "b200_pack_w4")
    return _packed(fmt, K, N, blob, K if group == -1 else group, int(n), perm is not None)


def pack_w8(q: torch.Tensor, col_scale: torch.Tensor) -> PackedWeight:
    _cuda_contig(q, col_scale)
    K, N = q.shape
    n = _lib.load().b200_wo_gemm_packed_bytes(B200_FMT_INT8, K, N)
    if n == 0:
        raise B200Error(f"pack_w8: unsupported shape K={K} N={N}")
    blob = _blob(int(n), K, None, q.device)
    check(_lib.load().b200_pack_w8(_p(q), K, N, _p(blob), _stream()), "b200_pack_w8")
    PackedWeight._write_trailer(blob, B200_FMT_INT8, K, N, 0)
    return PackedWeight(B200_FMT_INT8, K, N, blob, col_scale)


def pack_w8g(q: torch.Tensor, scales: torch.Tensor, zeros_x_scales: torch.Tensor, group: int = 128,
             perm: Optional[torch.Tensor] = None) -> PackedWeight:
    """8-bit group-wise (GPTQ/AWQ W8): q int8 [K,N] (q_s = q_u - 128), scales / zeros_x_scales [K/g,N] in the activation dtype.
    perm: as for pack_w4."""
    _cuda_contig(q, scales, zeros_x_scales)
    K, N = q.shape
    n = _lib.load().b200_wo_gemm_packed_bytes(B200_FMT_INT8G, K, N)
    if n == 0:
        raise B200Error(f"pack_w8g: unsupported shape K={K} N={N}")
    blob = _blob(int(n), K, perm, q.device)
    check(_lib.load().b200_pack_w8g(_p(q), _p(scales), _p(zeros_x_scales), K, N, group, _p(blob), _stream()), "b200_pack_w8g")
    return _packed(B200_FMT_INT8G, K, N, blob, group, int(n), perm is not None)


def pack_f16(w_kn: torch.Tensor) -> PackedWeight:
    """Reference stores W [K,N]; the kernel wants K contiguous -> one transpose at load time."""
    K, N = w_kn.shape
    return PackedWeight(B200_FMT_F16, K, N, w_kn.t().contiguous())


def gemm_workspace(max_batch: int, shapes, device) -> torch.Tensor:
    """One zero-filled scratch buffer big enough for every (K, N) in `shapes` (used serially on one stream)."""
    n = max(int(_lib.load().b200_wo_gemm_workspace_bytes(max_batch, N, K)) for (K, N) in shapes)
    return torch.zeros(max(n, 256), dtype=torch.uint8, device=device)


def gate_up_order(inter: int, device=None) -> torch.Tensor:
    """Column order that puts gate j and up j into ADJACENT rows of a 128-feature tile (row 2i = gate tile*64+i, row 2i+1 =
    up tile*64+i): the layout the fused SiLU*mul epilogue (B200_GEMM_SILU_MUL) expects of a [K, 2*inter] gate|up weight --
    the two values of a pair then sit in neighbouring lanes of one warp and are exchanged with a shuffle."""
    assert inter % 64 == 0
    j = torch.arange(inter, device=device)
    return torch.stack([j, j + inter], dim=1).reshape(-1)


def permute_columns(w: torch.Tensor, order: torch.Tensor, packed_int4: bool = False) -> torch.Tensor:
    """Column j of the result = column order[j] of w ([K, N], or uint8 [K, N/2] packed int4 -- low nibble = even column --, or
    scales [G, N] / [N])."""
    order = order.to(w.device)
    if packed_int4:
        full = torch.stack([w & 0xF, w >> 4], dim=-1).reshape(w.shape[0], -1)       # one nibble per column [K, N]
        full = full.index_select(-1, order)
        return (full[:, 0::2] | (full[:, 1::2] << 4)).contiguous()
    return w.index_select(-1, order).contiguous()


def interleave_gate_up(w: torch.Tensor, inter: int, packed_int4: bool = False) -> torch.Tensor:
    """Apply gate_up_order to the column axis of a reference-layout tensor (see permute_columns for the layouts)."""
    return permute_columns(w, gate_up_order(inter, w.device), packed_int4)


def reference_columns(fmt: str, w: torch.Tensor, scales: Optional[torch.Tensor] = None,
                      zeros_x_scales: Optional[torch.Tensor] = None, gate_up_inter: int = 0, col_perm: Optional[torch.Tensor] = None):
    """(w, scales, zeros_x_scales) of a reference-layout weight (see pack_reference) with its columns in packing order.
    col_perm: the row order of the w2 that consumes this gate|up weight's SiLU*mul output (an act-order w2, rows sorted by
    g_idx), folded into each half of the columns: gate and up column j move to col_perm[j] of their half, so the GEMM emits
    act[:, col_perm] and the sorted w2 needs no gather. col_perm is extended with the identity up to the half: padded inter
    columns keep their place. gate_up_inter > 0: then gate and up are interleaved (interleave_gate_up)."""
    packed_int4 = fmt == "int4"
    ts = [w, scales, zeros_x_scales]
    orders = []
    if col_perm is not None:
        half = w.shape[1] * (2 if packed_int4 else 1) // 2
        cp = torch.cat([col_perm, torch.arange(col_perm.numel(), half, device=col_perm.device)])
        orders.append(torch.cat([cp, cp + half]))
    if gate_up_inter:
        orders.append(gate_up_order(gate_up_inter, w.device))
    for order in orders:
        ts = [None if t is None else permute_columns(t, order, packed_int4 and i == 0) for i, t in enumerate(ts)]
    return tuple(ts)


def pack_reference(fmt: str, w: torch.Tensor, scales: Optional[torch.Tensor] = None, zeros_x_scales: Optional[torch.Tensor] = None,
                   group: int = 128, gate_up_inter: int = 0, perm: Optional[torch.Tensor] = None,
                   col_perm: Optional[torch.Tensor] = None) -> PackedWeight:
    """A weight in the reference's [K, N] layout, on the device, packed for wo_gemm. fmt "int4": w uint8 [K, N/2] packed
    nibbles, scales / zeros_x_scales [K/group, N] (pack_w4); "int8g": w int8 [K, N] (pack_w8g); "int8": w int8 [K, N],
    scales the per-column scale [N] (pack_w8); "f16": w [K, N] (pack_f16). gate_up_inter / col_perm: the column order of a
    gate|up weight (reference_columns). perm: the act-order row order the blob carries (int4 / int8g)."""
    w, scales, zeros_x_scales = reference_columns(fmt, w, scales, zeros_x_scales, gate_up_inter, col_perm)
    if fmt in ("int4", "int8g"):
        return (pack_w4 if fmt == "int4" else pack_w8g)(w.contiguous(), scales.contiguous(), zeros_x_scales.contiguous(), group,
                                                        perm=perm)
    if fmt == "int8":
        return pack_w8(w.contiguous(), scales.contiguous())
    if fmt == "f16":
        return pack_f16(w)
    raise B200Error(f"pack_reference: unknown weight format {fmt!r} (int4, int8g, int8 or f16)")


def permute_cols(x: torch.Tensor, perm: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[r][j] = x[r][perm[j]] (x [rows, K] fp16 / bf16, perm int32 [K] on the device): a bit copy."""
    _cuda_contig(x, perm, out)
    rows, K = x.shape
    _need("permute_cols", "perm", perm, torch.int32, (K,), flat=True)
    if out is None:
        out = torch.empty_like(x)
    if out.shape != x.shape or out.dtype != x.dtype:
        raise B200Error(f"permute_cols: out {tuple(out.shape)} {out.dtype} does not match x {tuple(x.shape)} {x.dtype}")
    check(_lib.load().b200_permute_cols(_p(x), _p(perm), _p(out), _is_bf16(x), rows, K, _stream()), "b200_permute_cols")
    return out


def wo_gemm(x: torch.Tensor, w: PackedWeight, workspace: torch.Tensor, bias: Optional[torch.Tensor] = None,
            out: Optional[torch.Tensor] = None, pdl: bool = False, silu_mul: bool = False,
            x_perm: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = x . W (+ bias). An act-order weight (w.perm set) needs x_perm, a scratch [>= B, K] of x's dtype: x[:, w.perm] is
    gathered into it (b200_permute_cols) and the GEMM reads that. bias: [N] of x's dtype; out: [B, N] ([B, N/2] with
    silu_mul) of x's dtype."""
    _cuda_contig(x, w.data, workspace, bias, out)
    B, K = x.shape
    if K != w.K:
        raise B200Error(f"wo_gemm: x has K={K}, weight has K={w.K}")
    n_out = w.N // 2 if silu_mul else w.N
    if bias is not None and (bias.dtype != x.dtype or tuple(bias.shape) != (w.N,)):
        raise B200Error(f"wo_gemm: bias must be [{w.N}] {x.dtype}, got {list(bias.shape)} {bias.dtype}")
    if out is not None and (out.dtype != x.dtype or tuple(out.shape) != (B, n_out)):
        raise B200Error(f"wo_gemm: out must be [{B}, {n_out}] {x.dtype}, got {list(out.shape)} {out.dtype}")
    if w.perm is not None:
        if x_perm is None:
            raise B200Error("wo_gemm: the weight is act-order (rows sorted by g_idx): pass x_perm, a [>= B, K] scratch for x[:, perm]")
        if x_perm.dim() != 2 or x_perm.shape[0] < B or x_perm.shape[1] != K or x_perm.dtype != x.dtype:
            raise B200Error(f"wo_gemm: x_perm must be [>= {B}, {K}] {x.dtype}, got {tuple(x_perm.shape)} {x_perm.dtype}")
        x = permute_cols(x, w.perm, out=x_perm[:B])
    if out is None:
        out = torch.empty((B, n_out), dtype=x.dtype, device=x.device)
    check(_lib.load().b200_wo_gemm(w.fmt, _is_bf16(x), _p(x), B, K, w.N, _p(w.data), _p(w.col_scale), _p(bias), _p(out),
                                   _p(workspace), workspace.numel(),
                                   (_lib.B200_GEMM_PDL if pdl else 0) | (_lib.B200_GEMM_SILU_MUL if silu_mul else 0), _stream()),
          "b200_wo_gemm")
    return out


# ------------------------------------------------------------------------------------------------ glue ops
def add_rmsnorm(x, residual, gamma, eps, out=None):
    _cuda_contig(x, residual, gamma, out)
    rows, hidden = x.shape
    if out is None:
        out = torch.empty_like(x)
    check(_lib.load().b200_add_rmsnorm(_p(x), _p(residual), _p(gamma), _p(out), _is_bf16(x), rows, hidden, eps, _stream()),
          "b200_add_rmsnorm")
    return out


def qk_rmsnorm(qkv, q_gamma, k_gamma, head_num, kv_head_num, head_dim, eps, q_bias=None, k_bias=None):
    """In-place per-head RMSNorm of the q and k heads of qkv [rows, (Hq+2Hkv)*D] (fused_qk_rmsnorm.cu)."""
    _cuda_contig(qkv, q_gamma, k_gamma, q_bias, k_bias)
    check(_lib.load().b200_qk_rmsnorm(_p(qkv), _p(q_gamma), _p(k_gamma), _p(q_bias), _p(k_bias), _is_bf16(qkv), qkv.shape[0], head_num,
                                      kv_head_num, head_dim, eps, _stream()), "b200_qk_rmsnorm")
    return qkv


def silu_and_mul(gate_up, out=None):
    _cuda_contig(gate_up, out)
    rows, two_inter = gate_up.shape
    if out is None:
        out = torch.empty((rows, two_inter // 2), dtype=gate_up.dtype, device=gate_up.device)
    check(_lib.load().b200_silu_and_mul(_p(gate_up), _p(out), _is_bf16(gate_up), rows, two_inter // 2, _stream()),
          "b200_silu_and_mul")
    return out


def _rope_args(what, qkv, kv_cache_base, page_list, sequence_lengths, head_num, q_out, q_len, qk_norm=None, bias=None,
               rope_cfg=None, position_ids=None, cos_sin_cache=None, use_logn_attn=False):
    """Checks and C arguments shared by the four rope + append ops: (q_out, (q_out, pool, page list, sequence lengths),
    the _ex entries' (position ids, table, table positions, config, logn), (dtype, B, Hq, Hkv, D, max blocks, page size)).
    qk_norm: (q_gamma, k_gamma), each a [D] tensor of qkv's dtype."""
    _cuda_contig(qkv, kv_cache_base, page_list, q_out, bias, position_ids, cos_sin_cache, *(qk_norm or ()))
    P, two, Hkv, T, D = kv_cache_base.shape
    rows = qkv.shape[0]
    if q_len < 1 or rows % q_len:
        raise B200Error(f"{what}: {rows} qkv rows are not a multiple of q_len {q_len}")
    check_lengths(what, sequence_lengths, rows // q_len)
    if position_ids is not None and position_ids.numel() != rows:
        raise B200Error(f"{what}: {position_ids.numel()} position ids for {rows} qkv rows")
    for name, g in zip(("q_gamma", "k_gamma"), qk_norm or ()):
        if g is None or g.dtype != qkv.dtype or g.numel() != D:
            raise B200Error(f"{what}: {name} must be a [{D}] tensor of qkv's dtype {qkv.dtype}")
    if q_out is None:
        q_out = torch.empty((rows, head_num * D), dtype=qkv.dtype, device=qkv.device)
    ex = ()
    if rope_cfg is not None:
        import ctypes
        ex = (_p(position_ids), _p(cos_sin_cache), cos_sin_cache.shape[0] if cos_sin_cache is not None else 0,
              ctypes.cast(ctypes.pointer(rope_cfg), ctypes.c_void_p), 1 if use_logn_attn else 0)
    return (q_out, (_p(q_out), _p(kv_cache_base), _p(page_list), _p(sequence_lengths)), ex,
            (_is_bf16(qkv), rows // q_len, head_num, Hkv, D, page_list.shape[-1], T))


def rope_append(qkv, kv_cache_base, page_list, sequence_lengths, head_num, rope_base, q_out=None, q_len: int = 1):
    """qkv [B*q_len, (Hq+2Hkv)*D]: q_len new tokens per sequence (row b*q_len + j = token j of sequence b, rotated and
    appended at sequence_lengths[b] + j). Returns q [B*q_len, Hq*D]."""
    q_out, io, _, shape = _rope_args("rope_append", qkv, kv_cache_base, page_list, sequence_lengths, head_num, q_out, q_len)
    lib = _lib.load()
    if q_len == 1:
        check(lib.b200_rope_append(_p(qkv), *io, *shape, rope_base, _stream()), "b200_rope_append")
    else:
        check(lib.b200_rope_append_multi(_p(qkv), *io, *shape, rope_base, q_len, _stream()), "b200_rope_append_multi")
    return q_out


def rope_append_ex(qkv, kv_cache_base, page_list, sequence_lengths, head_num, rope_cfg: "_lib.RopeConfig", q_out=None, bias=None,
                   position_ids=None, cos_sin_cache=None, use_logn_attn=False, q_len: int = 1):
    """FusedRopeKVCacheDecodeOp.forward with the whole rope contract (styles, position_ids override, bias, cos/sin cache,
    logn): see b200_rope_append_ex in include/b200_decode_ops.h. cos_sin_cache: fp32 [positions, dim] interleaved (cos, sin).
    q_len > 1: qkv [B*q_len, ...] holds q_len new tokens per sequence (row b*q_len + j = token j of sequence b, appended at
    sequence_lengths[b] + j) and position_ids, when given, has one entry per row. Returns q [B*q_len, Hq*D]."""
    q_out, io, ex, shape = _rope_args("rope_append_ex", qkv, kv_cache_base, page_list, sequence_lengths, head_num, q_out, q_len,
                                      bias=bias, rope_cfg=rope_cfg, position_ids=position_ids, cos_sin_cache=cos_sin_cache,
                                      use_logn_attn=use_logn_attn)
    lib = _lib.load()
    if q_len == 1:
        check(lib.b200_rope_append_ex(_p(qkv), _p(bias), *io, *ex, *shape, _stream()), "b200_rope_append_ex")
    else:
        check(lib.b200_rope_append_ex_multi(_p(qkv), _p(bias), *io, *ex, *shape, q_len, _stream()), "b200_rope_append_ex_multi")
    return q_out


def qk_norm_rope_append(qkv, q_gamma, k_gamma, eps, kv_cache_base, page_list, sequence_lengths, head_num, rope_base, q_out=None,
                        q_len: int = 1):
    """rope_append after Qwen3's QK-RMSNorm, in one launch: each q and k head of qkv is RMS-normalised with q_gamma / k_gamma
    [D] first, with the bits of qk_rmsnorm on a copy of qkv followed by rope_append (b200_qk_norm_rope_append). qkv is only
    read. Returns q [B*q_len, Hq*D]."""
    q_out, io, _, shape = _rope_args("qk_norm_rope_append", qkv, kv_cache_base, page_list, sequence_lengths, head_num, q_out, q_len,
                                     qk_norm=(q_gamma, k_gamma))
    check(_lib.load().b200_qk_norm_rope_append(_p(qkv), _p(q_gamma), _p(k_gamma), eps, *io, *shape, rope_base, q_len, _stream()),
          "b200_qk_norm_rope_append")
    return q_out


def qk_norm_rope_append_ex(qkv, q_gamma, k_gamma, eps, kv_cache_base, page_list, sequence_lengths, head_num,
                           rope_cfg: "_lib.RopeConfig", q_out=None, position_ids=None, cos_sin_cache=None, use_logn_attn=False,
                           q_len: int = 1):
    """rope_append_ex (no bias) after Qwen3's QK-RMSNorm, in one launch (b200_qk_norm_rope_append_ex): the bits of qk_rmsnorm
    on a copy of qkv followed by rope_append_ex. qkv is only read. Returns q [B*q_len, Hq*D]."""
    q_out, io, ex, shape = _rope_args("qk_norm_rope_append_ex", qkv, kv_cache_base, page_list, sequence_lengths, head_num, q_out,
                                      q_len, qk_norm=(q_gamma, k_gamma), rope_cfg=rope_cfg, position_ids=position_ids,
                                      cos_sin_cache=cos_sin_cache, use_logn_attn=use_logn_attn)
    check(_lib.load().b200_qk_norm_rope_append_ex(_p(qkv), _p(q_gamma), _p(k_gamma), eps, *io, *ex, *shape, q_len, _stream()),
          "b200_qk_norm_rope_append_ex")
    return q_out


def embedding(ids, table, out=None):
    _cuda_contig(ids, table, out)
    rows, hidden = ids.shape[0], table.shape[1]
    if out is None:
        out = torch.empty((rows, hidden), dtype=table.dtype, device=table.device)
    check(_lib.load().b200_embedding(_p(ids), _p(table), _p(out), _is_bf16(table), rows, hidden, _stream()), "b200_embedding")
    return out


def argmax(logits, out=None):
    dt = _logit_dtype("argmax", logits)
    _cuda_contig(logits, out)
    rows, vocab = logits.shape
    if out is None:
        out = torch.empty(rows, dtype=torch.int32, device=logits.device)
    check(_lib.load().b200_argmax(_p(logits), dt, rows, vocab, _p(out), _stream()), "b200_argmax")
    return out


def sample(logits: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor, uniform: torch.Tensor,
           temperature: Optional[torch.Tensor] = None, history: Optional[torch.Tensor] = None,
           hist_len: Optional[torch.Tensor] = None, repetition: Optional[torch.Tensor] = None,
           presence: Optional[torch.Tensor] = None, frequency: Optional[torch.Tensor] = None,
           process: Optional[torch.Tensor] = None, count_ws: Optional[torch.Tensor] = None, want_probs: bool = False,
           out: Optional[dict] = None, min_p: Optional[torch.Tensor] = None):
    """sampleGreedy's CUDA path (CudaSampleOp.cc:423-463) on fp32 logits [B, V], IN PLACE (logits become probabilities).
    Returns (tokens int32 [B], token_prob fp32 [B], renormalised probs [B, V] or None). `out` may hold preallocated
    token int32 [B], token_prob fp32 [B] and probs fp32 [B, V] (graph capture); a given probs implies want_probs.
    min_p fp32 [B] in [0, 1] (None: off) keeps only p >= min_p * p_max of what top-k / top-p keep; its range is checked on the
    host (a device read) except while a CUDA graph is being captured, where the kernel clamps it."""
    B, V = logits.shape
    probs = dict(probs=(torch.float32, (B, V))) if want_probs or (out or {}).get("probs") is not None else {}
    out = _outputs("sample", out, logits.device, token=(torch.int32, (B,)), token_prob=(torch.float32, (B,)), **probs)
    if min_p is not None:
        _need("sample", "min_p", min_p, torch.float32, (B,), flat=True)
        capturing = min_p.is_cuda and torch.cuda.is_current_stream_capturing()
        if not capturing and not bool(((min_p >= 0) & (min_p <= 1)).all()):
            raise B200Error("sample: min_p must be in [0, 1]")
    _cuda_contig(logits, top_k, top_p, uniform, temperature, history, hist_len, repetition, presence, frequency, process, count_ws,
                 min_p, *out.values())
    if logits.dtype != torch.float32:
        raise B200Error("sample: logits must be fp32 (the reference sampler runs on fp32 logits)")
    if (repetition is not None or presence is not None or frequency is not None) and count_ws is None:
        count_ws = torch.zeros(B, V, dtype=torch.int32, device=logits.device)
    check(_lib.load().b200_sample(_p(logits), B, V, _p(history), _p(hist_len), history.shape[1] if history is not None else 0,
                                  _p(count_ws), _p(temperature), _p(repetition), _p(presence), _p(frequency), _p(top_k), _p(top_p),
                                  _p(min_p), _p(uniform), _p(process), _p(out["token"]), _p(out["token_prob"]), _p(out.get("probs")),
                                  _stream()), "b200_sample")
    return out["token"], out["token_prob"], out.get("probs")


def _spec_verify_args(who: str, device, B: int, nodes: int, draft_rows: int, target_probs, target_ids, uniform, draft_probs,
                      outs: dict):
    """The checks and outputs both verification wrappers share, for B sequences of `nodes` rows: the greedy (target_ids) or
    sampling (target_probs, uniform) inputs, draft_probs [B, draft_rows, V] in sampling mode, and the outputs of `outs` (name:
    tensor or None), out_tokens [B, nodes], accepted [B] and accepted_path [B, nodes]. Returns (V, outputs)."""
    if target_probs is None and target_ids is None:
        raise B200Error(f"{who}: pass target_probs (sampling) or target_ids (greedy)")
    if target_probs is not None:
        _need(who, "target_probs", target_probs, torch.float32, (B, nodes, "V"))
        V = target_probs.shape[2]
        if uniform is None or uniform.dtype != torch.float32 or uniform.numel() != B * nodes:
            raise B200Error(f"{who}: sampling mode needs uniform fp32 [{B}, {nodes}]")
        if draft_probs is not None:
            _need(who, "draft_probs", draft_probs, torch.float32, (B, draft_rows, V))
    else:
        _need(who, "target_ids", target_ids, torch.int32, (B, nodes))
        V = 1                                   # the vocabulary is not read in greedy mode
    shapes = dict(out_tokens=(torch.int32, (B, nodes)), accepted=(torch.int32, (B,)), accepted_path=(torch.int32, (B, nodes)))
    return V, _outputs(who, outs, device, **{k: shapes[k] for k in outs})


def spec_verify(draft_tokens: torch.Tensor, *, target_probs: Optional[torch.Tensor] = None,
                target_ids: Optional[torch.Tensor] = None, draft_probs: Optional[torch.Tensor] = None,
                uniform: Optional[torch.Tensor] = None, out_tokens: Optional[torch.Tensor] = None,
                accepted: Optional[torch.Tensor] = None):
    """Verify n = draft_tokens.shape[1] speculative tokens per sequence (b200_spec_verify). Greedy: target_ids int32 [B, n+1]
    (argmax of the step's rows). Sampling: target_probs fp32 [B, n+1, V], optional draft_probs fp32 [B, n, V] (None =
    deterministic drafts), uniform fp32 [B, n+1]. Returns (out_tokens int32 [B, n+1]: accepted drafts, then one correction or
    bonus token, then -1; accepted int32 [B])."""
    _cuda_contig(draft_tokens, target_probs, target_ids, draft_probs, uniform, out_tokens, accepted)
    B, n = draft_tokens.shape
    V, out = _spec_verify_args("spec_verify", draft_tokens.device, B, n + 1, n, target_probs, target_ids, uniform, draft_probs,
                               dict(out_tokens=out_tokens, accepted=accepted))
    if draft_tokens.dtype != torch.int32:
        raise B200Error("spec_verify: draft_tokens must be int32")
    check(_lib.load().b200_spec_verify(_p(target_probs), _p(target_ids), _p(draft_probs), _p(draft_tokens), _p(uniform), B, n, V,
                                       _p(out["out_tokens"]), _p(out["accepted"]), _stream()), "b200_spec_verify")
    return out["out_tokens"], out["accepted"]


def spec_verify_tree_draft_workspace(batch: int, vocab: int, device) -> torch.Tensor:
    """Workspace of b200_spec_verify_tree_draft (the residual rows; no initial contents needed)."""
    n = int(_lib.load().b200_spec_verify_tree_draft_workspace_bytes(batch, vocab))
    return torch.empty(max(n, 16), dtype=torch.uint8, device=device)


def spec_verify_tree(tree_parents: torch.Tensor, node_tokens: torch.Tensor, *, target_probs: Optional[torch.Tensor] = None,
                     target_ids: Optional[torch.Tensor] = None, uniform: Optional[torch.Tensor] = None,
                     out_tokens: Optional[torch.Tensor] = None, accepted: Optional[torch.Tensor] = None,
                     accepted_path: Optional[torch.Tensor] = None, draft_probs: Optional[torch.Tensor] = None,
                     workspace: Optional[torch.Tensor] = None):
    """Verify a speculative token tree of n = tree_parents.shape[1] <= 64 nodes per sequence (b200_spec_verify_tree).
    tree_parents, node_tokens int32 [B, n] (node 0 the root; its token is not read). Greedy: target_ids int32 [B, n]. Sampling
    (deterministic drafts): target_probs fp32 [B, n, V], uniform fp32 [B, n]. Sampling with draft_probs fp32 [B, n, V] (row c:
    the distribution node c's token was drawn from; n >= 2): recursive rejection (b200_spec_verify_tree_draft), in `workspace`
    (spec_verify_tree_draft_workspace; allocated when not given). Returns (out_tokens int32 [B, n]: the accepted path's tokens,
    then one correction or bonus token, then -1; accepted int32 [B]; accepted_path int32 [B, n]: the node at depth 0 ..
    accepted, then -1)."""
    if draft_probs is not None and target_probs is None:
        raise B200Error("spec_verify_tree: draft_probs need the sampling mode (target_probs)")
    _cuda_contig(tree_parents, node_tokens, target_probs, target_ids, uniform, out_tokens, accepted, accepted_path, draft_probs,
                 workspace)
    if tree_parents.dim() != 2:
        raise B200Error("spec_verify_tree: tree_parents must be [B, n]")
    B, n = tree_parents.shape
    if tree_parents.dtype != torch.int32 or node_tokens.dtype != torch.int32 or tuple(node_tokens.shape) != (B, n):
        raise B200Error(f"spec_verify_tree: tree_parents and node_tokens must be int32 [{B}, {n}]")
    V, out = _spec_verify_args("spec_verify_tree", tree_parents.device, B, n, n, target_probs, target_ids, uniform, draft_probs,
                               dict(out_tokens=out_tokens, accepted=accepted, accepted_path=accepted_path))
    outs = (_p(out["out_tokens"]), _p(out["accepted"]), _p(out["accepted_path"]), _stream())
    if draft_probs is None:
        check(_lib.load().b200_spec_verify_tree(_p(target_probs), _p(target_ids), _p(tree_parents), _p(node_tokens), _p(uniform), B, n,
                                                V, *outs), "b200_spec_verify_tree")
        return out["out_tokens"], out["accepted"], out["accepted_path"]
    need = int(_lib.load().b200_spec_verify_tree_draft_workspace_bytes(B, V))
    if workspace is None:
        workspace = spec_verify_tree_draft_workspace(B, V, tree_parents.device)
    elif workspace.dtype != torch.uint8 or workspace.numel() < need:
        raise B200Error(f"spec_verify_tree: workspace must be uint8 of at least {need} bytes (spec_verify_tree_draft_workspace)")
    check(_lib.load().b200_spec_verify_tree_draft(_p(target_probs), _p(draft_probs), _p(tree_parents), _p(node_tokens), _p(uniform),
                                                  B, n, V, _p(workspace), workspace.numel(), *outs), "b200_spec_verify_tree_draft")
    return out["out_tokens"], out["accepted"], out["accepted_path"]


def kv_compact_path(kv_caches: Sequence[torch.Tensor], page_list: torch.Tensor, sequence_lengths: torch.Tensor,
                    accepted_path: torch.Tensor, accepted: torch.Tensor) -> None:
    """Move the accepted path of a token-tree step to consecutive cache slots, in place, in one launch for every layer
    (b200_kv_compact_path): for d = 1 .. accepted[b] the K/V of slot sequence_lengths[b] + accepted_path[b][d] go to slot
    sequence_lengths[b] + d. kv_caches: one [P, 2, Hkv, T, D] cache per layer (fp16 / bf16, the same shape); page_list
    [B, 1, 2, M]; sequence_lengths, accepted int32 [B]; accepted_path int32 [B, n]."""
    kv_caches = list(kv_caches)
    if not kv_caches:
        raise B200Error("kv_compact_path: no layer caches given")
    _cuda_contig(*kv_caches, page_list, sequence_lengths, accepted_path, accepted)
    shape = tuple(kv_caches[0].shape)
    if len(shape) != 5 or any(tuple(c.shape) != shape or c.dtype != kv_caches[0].dtype for c in kv_caches):
        raise B200Error("kv_compact_path: every layer cache must be [P, 2, Hkv, T, D] of one shape and dtype")
    _is_bf16(kv_caches[0])
    P, two, Hkv, T, D = shape
    if accepted_path.dim() != 2:
        raise B200Error("kv_compact_path: accepted_path must be [B, n]")
    B, n = accepted_path.shape
    _need("kv_compact_path", "sequence_lengths", sequence_lengths, torch.int32, (B,))
    _need("kv_compact_path", "accepted", accepted, torch.int32, (B,))
    _need("kv_compact_path", "accepted_path", accepted_path, torch.int32, (B, n))
    if page_list.dtype != torch.int32 or page_list.dim() != 4 or page_list.shape[0] != B:
        raise B200Error(f"kv_compact_path: page_list must be int32 [{B}, 1, 2, M]")
    import ctypes
    pools = (ctypes.c_void_p * len(kv_caches))(*[c.data_ptr() for c in kv_caches])
    check(_lib.load().b200_kv_compact_path(pools, len(kv_caches), Hkv, D, T, _p(page_list), page_list.shape[-1], _p(sequence_lengths),
                                           _p(accepted_path), _p(accepted), B, n, _stream()), "b200_kv_compact_path")


_LOGIT_DTYPES = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


def _logit_dtype(who: str, logits: torch.Tensor) -> int:
    if logits.dtype not in _LOGIT_DTYPES:
        raise B200Error(f"{who}: logits must be fp16, bf16 or fp32 (got {logits.dtype})")
    return _LOGIT_DTYPES[logits.dtype]


def beam_search_workspace(batch: int, beam_width: int, vocab: int, device) -> torch.Tensor:
    """Zeroed workspace of b200_beam_search_step for up to `batch` requests (its counters reset themselves after every call)."""
    n = int(_lib.load().b200_beam_search_step_workspace_bytes(batch, beam_width, vocab))
    if n == 0:
        raise B200Error(f"beam_search_step: unsupported shape batch {batch}, beam_width {beam_width}, vocab {vocab}")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def beam_search_step(logits: torch.Tensor, cum_log_probs: torch.Tensor, beam_width: int, eos_id: int = -1,
                     workspace: Optional[torch.Tensor] = None, out: Optional[dict] = None) -> dict:
    """One beam-search step (b200_beam_search_step): logits [B*W, V] fp16 / bf16 / fp32 (row b*W + i = beam i of request b),
    cum_log_probs fp32 [B, W]. Returns dict(cand_token, cand_parent, cand_score [B, 2W]: the top 2W candidates in rank order;
    next_token, next_parent, next_cum [B, W]: the first W of them whose token is not eos_id). `out` may hold those six
    tensors preallocated (graph capture); `workspace` comes from beam_search_workspace."""
    W = beam_width
    if not 1 <= W <= 32:
        raise B200Error(f"beam_search_step: beam_width {W} unsupported (1..32)")
    if logits.dim() != 2 or logits.shape[0] % W:
        raise B200Error(f"beam_search_step: logits must be [B * {W}, V] (got {tuple(logits.shape)})")
    dt = _logit_dtype("beam_search_step", logits)
    rows, V = logits.shape
    B = rows // W
    if V < 2 * W:
        raise B200Error(f"beam_search_step: vocab {V} must be >= 2 * beam_width ({2 * W})")
    _need("beam_search_step", "cum_log_probs", cum_log_probs, torch.float32, (B, W), flat=True)
    shapes = dict(cand_token=(torch.int32, (B, 2 * W)), cand_parent=(torch.int32, (B, 2 * W)), cand_score=(torch.float32, (B, 2 * W)),
                  next_token=(torch.int32, (B, W)), next_parent=(torch.int32, (B, W)), next_cum=(torch.float32, (B, W)))
    out = _outputs("beam_search_step", out, logits.device, **shapes)
    if workspace is None:
        workspace = beam_search_workspace(B, W, V, logits.device)
    _cuda_contig(logits, cum_log_probs, workspace, *out.values())
    check(_lib.load().b200_beam_search_step(_p(logits), dt, _p(cum_log_probs), B, W, V, eos_id, *(_p(out[k]) for k in shapes),
                                            _p(workspace), workspace.numel(), _stream()), "b200_beam_search_step")
    return out


def beam_hypotheses_state(batch: int, beam_width: int, max_len: int, device) -> torch.Tensor:
    """Empty finished-hypothesis sets (all-zero bytes) of `batch` requests, W = beam_width slots of up to max_len tokens each:
    the state of beam_hypotheses_update / beam_hypotheses_finalize (layout in include/b200_decode_ops.h). zero_() restarts it."""
    n = int(_lib.load().b200_beam_hypotheses_state_bytes(batch, beam_width, max_len))
    if n == 0 and batch != 0:
        raise B200Error(f"beam_hypotheses: unsupported shape batch {batch}, beam_width {beam_width}, max_len {max_len}")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def _beam_hyps_checks(who: str, B: int, W: int, max_len: int, history, hist_len, length_penalty, state, done) -> None:
    if not 1 <= W <= 32:
        raise B200Error(f"{who}: beam_width {W} unsupported (1..32)")
    if history.dtype != torch.int32 or history.dim() != 2 or history.shape[0] != B * W or history.shape[1] < 1:
        raise B200Error(f"{who}: history must be int32 [{B * W}, stride >= 1]")
    _need(who, "hist_len", hist_len, torch.int32, (B * W,), flat=True)
    _need(who, "length_penalty", length_penalty, torch.float32, (B,), flat=True)
    _need(who, "done", done, torch.int32, (B,), flat=True)
    need = int(_lib.load().b200_beam_hypotheses_state_bytes(B, W, max_len))
    if state.dtype != torch.uint8 or (need == 0 and B != 0) or state.numel() < need:
        raise B200Error(f"{who}: state must be uint8 of at least {need} bytes (beam_hypotheses_state({B}, {W}, {max_len}))")


def beam_hypotheses_update(beam_out: dict, history: torch.Tensor, hist_len: torch.Tensor, eos_id: int, length_penalty: torch.Tensor,
                           early_stopping: torch.Tensor, state: torch.Tensor, done: torch.Tensor, max_len: int,
                           gen_start: int = 0) -> None:
    """b200_beam_hypotheses_update, after beam_search_step and before the fork: the EOS candidates among the first W ranks of
    beam_out (beam_search_step's cand_token / cand_parent / cand_score [B, 2W]) enter each request's finished set in `state`
    (beam_hypotheses_state(B, W, max_len)), with the path history[B*W, stride][gen_start : hist_len] + eos_id. length_penalty
    fp32 [B]; early_stopping int32 [B] (0 False, 1 True, 2 "never"); done int32 [B] is set once a request is done, and a done
    request is left alone."""
    ct = beam_out["cand_token"]
    if ct.dim() != 2 or ct.shape[1] % 2:
        raise B200Error(f"beam_hypotheses_update: cand_token must be [B, 2W] (got {tuple(ct.shape)})")
    B, W = ct.shape[0], ct.shape[1] // 2
    _beam_hyps_checks("beam_hypotheses_update", B, W, max_len, history, hist_len, length_penalty, state, done)
    for k, dt in (("cand_token", torch.int32), ("cand_parent", torch.int32), ("cand_score", torch.float32)):
        if beam_out[k].dtype != dt or beam_out[k].numel() != B * 2 * W:
            raise B200Error(f"beam_hypotheses_update: {k} must be {dt} [{B}, {2 * W}]")
    _need("beam_hypotheses_update", "early_stopping", early_stopping, torch.int32, (B,), flat=True)
    if eos_id < 0:
        raise B200Error(f"beam_hypotheses_update: eos_id {eos_id} must be >= 0")
    _cuda_contig(ct, beam_out["cand_parent"], beam_out["cand_score"], history, hist_len, length_penalty, early_stopping, state, done)
    check(_lib.load().b200_beam_hypotheses_update(_p(ct), _p(beam_out["cand_parent"]), _p(beam_out["cand_score"]), _p(history),
                                                  _p(hist_len), history.shape[1], gen_start, B, W, eos_id, _p(length_penalty),
                                                  _p(early_stopping), max_len, _p(state), state.numel(), _p(done), _stream()),
          "b200_beam_hypotheses_update")


def beam_hypotheses_finalize(state: torch.Tensor, done: torch.Tensor, beam_cum: torch.Tensor, history: torch.Tensor,
                             hist_len: torch.Tensor, n: int, max_len: int, length_penalty: torch.Tensor, gen_start: int = 0,
                             out: Optional[dict] = None) -> dict:
    """b200_beam_hypotheses_finalize: the n (1..W) best hypotheses of each request, the live beams (beam_cum fp32 [B, W] and
    their history rows) merged in for a request that is not done. Returns dict(tokens int32 [B, n, max_len] (-1 past the
    path), len int32 [B, n], score fp32 [B, n] (cum / len^length_penalty, descending), cum fp32 [B, n]); a missing
    hypothesis has tokens and len -1, score and cum -inf. The state is not modified."""
    if beam_cum.dtype != torch.float32 or beam_cum.dim() != 2:
        raise B200Error(f"beam_hypotheses_finalize: beam_cum must be fp32 [B, W] (got {beam_cum.dtype} {tuple(beam_cum.shape)})")
    B, W = beam_cum.shape
    _beam_hyps_checks("beam_hypotheses_finalize", B, W, max_len, history, hist_len, length_penalty, state, done)
    if not 1 <= n <= W:
        raise B200Error(f"beam_hypotheses_finalize: n {n} unsupported (1..beam_width {W})")
    shapes = dict(tokens=(torch.int32, (B, n, max_len)), len=(torch.int32, (B, n)), score=(torch.float32, (B, n)),
                  cum=(torch.float32, (B, n)))
    out = _outputs("beam_hypotheses_finalize", out, beam_cum.device, **shapes)
    _cuda_contig(state, done, beam_cum, history, hist_len, length_penalty, *out.values())
    check(_lib.load().b200_beam_hypotheses_finalize(_p(state), state.numel(), _p(done), _p(beam_cum), _p(history), _p(hist_len),
                                                    history.shape[1], gen_start, B, W, n, max_len, _p(length_penalty),
                                                    *(_p(out[k]) for k in shapes), _stream()), "b200_beam_hypotheses_finalize")
    return out


LOGPROB_MAX_TOP_N = 64


def token_logprobs_workspace(rows: int, vocab: int, top_n: int, device) -> torch.Tensor:
    """Zeroed workspace of b200_token_logprobs (its counters reset themselves after every call)."""
    n = int(_lib.load().b200_token_logprobs_workspace_bytes(rows, vocab, top_n))
    if n == 0:
        raise B200Error(f"token_logprobs: unsupported shape rows {rows}, vocab {vocab}, top_n {top_n}")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def token_logprobs(logits: torch.Tensor, top_n: int = 0, tokens: Optional[torch.Tensor] = None,
                   workspace: Optional[torch.Tensor] = None, out: Optional[dict] = None) -> dict:
    """Log-probabilities of the raw lm_head output (b200_token_logprobs): logits [rows, V] fp16 / bf16 / fp32, log-softmax per row
    in fp32 before any temperature, penalty or filter. Returns dict(token_logprob fp32 [rows] = lp of tokens int32 [rows], when
    tokens is given; top_ids int32 / top_logprobs fp32 [rows, top_n]: the top_n largest, descending, equal values by lower id).
    top_n in 0..64 (and <= V, ceil(V / 4096) * top_n <= 4096). `out` may hold the output tensors preallocated (graph capture);
    `workspace` comes from token_logprobs_workspace."""
    dt = _logit_dtype("token_logprobs", logits)
    if logits.dim() != 2:
        raise B200Error(f"token_logprobs: logits must be [rows, V] (got {tuple(logits.shape)})")
    rows, V = logits.shape
    if not 0 <= top_n <= min(LOGPROB_MAX_TOP_N, V) or (V + 4095) // 4096 * top_n > 4096:
        raise B200Error(f"token_logprobs: top_n {top_n} unsupported (0..{LOGPROB_MAX_TOP_N}, <= vocab {V}, "
                        f"ceil(vocab / 4096) * top_n <= 4096)")
    token_logprob = {}
    if tokens is not None:
        _need("token_logprobs", "tokens", tokens, torch.int32, (rows,), flat=True)
        token_logprob = dict(token_logprob=(torch.float32, (rows,)))
    out = _outputs("token_logprobs", out, logits.device, top_ids=(torch.int32, (rows, top_n)),
                   top_logprobs=(torch.float32, (rows, top_n)), **token_logprob)
    need = int(_lib.load().b200_token_logprobs_workspace_bytes(rows, V, top_n))
    if workspace is None:
        workspace = token_logprobs_workspace(rows, V, top_n, logits.device)
    elif workspace.dtype != torch.uint8 or workspace.numel() < need:
        raise B200Error(f"token_logprobs: workspace must be uint8 of at least {need} bytes (token_logprobs_workspace)")
    _cuda_contig(logits, tokens, workspace, *out.values())
    check(_lib.load().b200_token_logprobs(_p(logits), dt, rows, V, top_n, _p(tokens), _p(out.get("token_logprob")),
                                          _p(out["top_ids"]), _p(out["top_logprobs"]), _p(workspace), workspace.numel(), _stream()),
          "b200_token_logprobs")
    return out


def ban_repeat_ngram(logits: torch.Tensor, history: torch.Tensor, hist_len: torch.Tensor, ngram_size: torch.Tensor) -> torch.Tensor:
    """No-repeat-n-gram ban in place (b200_ban_repeat_ngram): logits [rows, V] fp16 / bf16 / fp32, history int32
    [rows, stride], hist_len int32 [rows], ngram_size int32 [rows] (<= 0: off). Returns logits."""
    dt = _logit_dtype("ban_repeat_ngram", logits)
    if logits.dim() != 2:
        raise B200Error(f"ban_repeat_ngram: logits must be [rows, V] (got {tuple(logits.shape)})")
    rows, V = logits.shape
    if history.dtype != torch.int32 or history.dim() != 2 or history.shape[0] != rows or history.shape[1] < 1:
        raise B200Error(f"ban_repeat_ngram: history must be int32 [{rows}, stride >= 1]")
    _need("ban_repeat_ngram", "hist_len", hist_len, torch.int32, (rows,), flat=True)
    _need("ban_repeat_ngram", "ngram_size", ngram_size, torch.int32, (rows,), flat=True)
    _cuda_contig(logits, history, hist_len, ngram_size)
    check(_lib.load().b200_ban_repeat_ngram(_p(logits), dt, rows, V, _p(history), _p(hist_len), history.shape[1], _p(ngram_size),
                                            _stream()), "b200_ban_repeat_ngram")
    return logits


def constrain_logits(logits: torch.Tensor, bitmask: Optional[torch.Tensor] = None,
                     logit_bias: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
    """Grammar mask and logit bias in place (b200_constrain_logits): logits [rows, V] fp16 / bf16 / fp32; bitmask int32
    [rows, stride >= ceil(V / 32)] in xgrammar's layout (token t allowed iff bit t & 31 of word t >> 5 is set); logit_bias =
    (offsets int32 [rows + 1], ids int32 [n], values fp32 [n]), a CSR over rows with offsets[rows] <= n (logit_bias_csr builds
    it on the host; n = 0 is no bias, and without a bitmask then launches nothing). Masked tokens become -inf, allowed biased
    ones round(x + bias). Returns logits."""
    dt = _logit_dtype("constrain_logits", logits)
    if logits.dim() != 2:
        raise B200Error(f"constrain_logits: logits must be [rows, V] (got {tuple(logits.shape)})")
    rows, V = logits.shape
    if not 1 <= rows <= 65535:
        raise B200Error(f"constrain_logits: rows {rows} unsupported (1..65535)")
    if bitmask is None and logit_bias is None:
        raise B200Error("constrain_logits: pass a bitmask, a logit_bias or both")
    words = (V + 31) // 32
    if bitmask is not None and (bitmask.dtype != torch.int32 or bitmask.dim() != 2 or bitmask.shape[0] != rows
                                or bitmask.shape[1] < words):
        raise B200Error(f"constrain_logits: bitmask must be int32 [{rows}, stride >= {words}] (got {bitmask.dtype} "
                        f"{tuple(bitmask.shape)})")
    offsets = ids = values = None
    if logit_bias is not None:
        offsets, ids, values = logit_bias
        _need("constrain_logits", "bias offsets", offsets, torch.int32, (rows + 1,), flat=True)
        if ids.dtype != torch.int32 or values.dtype != torch.float32 or ids.numel() != values.numel():
            raise B200Error("constrain_logits: bias ids must be int32 and values fp32, of one length")
    _cuda_contig(logits, bitmask, offsets, ids, values)
    if ids is not None and ids.numel() == 0:          # no entries: no bias (an empty tensor has no data pointer to pass)
        if bitmask is None:
            return logits
        offsets = ids = values = None
    check(_lib.load().b200_constrain_logits(_p(logits), dt, rows, V, _p(bitmask), 0 if bitmask is None else bitmask.shape[1],
                                            _p(offsets), _p(ids), _p(values), _stream()), "b200_constrain_logits")
    return logits


def logit_bias_csr(per_row: Sequence[Mapping[int, float]], vocab: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """OpenAI-style logit_bias maps {token id: bias}, one per row, as the CSR constrain_logits takes: (offsets int32
    [rows + 1], ids int32, values fp32), on the host. Rejects ids outside [0, vocab) and values that are not numbers or are
    NaN; a mapping holds each id once, so the ids of a row are distinct."""
    offsets, ids, values = [0], [], []
    for r, m in enumerate(per_row):
        for t, b in m.items():
            if isinstance(t, bool) or not isinstance(t, numbers.Integral) or not 0 <= t < vocab:
                raise B200Error(f"logit_bias_csr: row {r}: token id {t!r} outside [0, {vocab})")
            if isinstance(b, bool) or not isinstance(b, numbers.Real) or math.isnan(b):
                raise B200Error(f"logit_bias_csr: row {r}: bias {b!r} of token {t} is not a number")
            ids.append(int(t))
            values.append(float(b))
        offsets.append(len(ids))
    return (torch.tensor(offsets, dtype=torch.int32), torch.tensor(ids, dtype=torch.int32),
            torch.tensor(values, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------ decode programs
class Program:
    """Recorded sequence of op calls (b200_program_*): `with prog.record(): <ops...>` then `prog.launch()` replays them
    with the GEMMs / norms / rope between two attention calls fused into one persistent kernel. Pointers are frozen at
    record time (like a CUDA-graph capture); launch() is itself graph-capturable."""

    def __init__(self):
        import ctypes
        self._h = ctypes.c_void_p()
        check(_lib.load().b200_program_create(ctypes.byref(self._h)), "b200_program_create")
        self._keep = []

    class _Rec:
        def __init__(self, prog):
            self.prog = prog

        def __enter__(self):
            check(_lib.load().b200_program_begin(self.prog._h), "b200_program_begin")
            return self.prog

        def __exit__(self, et, ev, tb):
            rc = _lib.load().b200_program_end(self.prog._h)
            if et is None:
                check(rc, "b200_program_end")
            return False

    def record(self):
        return Program._Rec(self)

    def launch(self) -> None:
        check(_lib.load().b200_program_launch(self._h, _stream()), "b200_program_launch")

    @property
    def num_ops(self) -> int:
        return int(_lib.load().b200_program_num_ops(self._h))

    @property
    def num_launches(self) -> int:
        return int(_lib.load().b200_program_num_launches(self._h))

    def set_trace(self, buf: Optional[torch.Tensor]) -> None:
        self._keep.append(buf)
        check(_lib.load().b200_program_set_trace(self._h, _p(buf)), "b200_program_set_trace")

    def __del__(self):
        try:
            if self._h:
                _lib.load().b200_program_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass
