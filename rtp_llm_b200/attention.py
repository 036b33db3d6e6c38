"""Host-side mirror of the reference's decode-attention seam, over the C ABI.

  B200DecodeAttnOp   == the pybind class XQAAttnOp (support / prepare / update / update_kv_cache_offset / forward),
                        /root/reference/rtp_llm/models_py/bindings/cuda/XQAAttnOp.{h:13-28,cc:52-176}
  B200DecodeImpl     == an FMHAImplBase strategy (ctor (attn_configs, attn_inputs, parallelism_config), static support,
                        forward(qkv, kv_cache, layer_idx), prepare_cuda_graph(attn_inputs)),
                        /root/reference/rtp_llm/models_py/modules/factory/attention/fmha_impl_base.py:99-175 and
                        cuda_impl/xqa.py:61-153 (the structure mirrored here: rope+append op, then the paged attention op)

Inside the reference tree the impl is appended to DECODE_MHA_IMPS (attention/__init__.py:91-100); see INTEGRATION.md.
Config / input objects are duck-typed: any object with the reference's attribute names works (AttentionConfigs:
head_num, kv_head_num, size_per_head, kernel_tokens_per_block|tokens_per_block, max_seq_len, need_rope_kv_cache,
rope_config (style, dim, base, scale, factor1, factor2, max_pos, extrapolation_factor, mscale, is_neox_style; see rope.py),
use_logn_attn, q_scaling; PyAttentionInputs: sequence_lengths, kv_cache_kernel_block_id_device, is_prefill, combo_position_ids
when the rotation positions are not the cache slots, and input_lengths for a verification step of speculative tokens, which
runs q_len = max(input_lengths) tokens per sequence).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from . import ops, rope
from ._lib import B200Error

try:  # inside the reference tree the real base class is used; standalone, a structural stand-in
    from rtp_llm.models_py.modules.factory.attention.fmha_impl_base import FMHAImplBase  # type: ignore
except Exception:  # noqa: BLE001
    class FMHAImplBase:  # same surface as fmha_impl_base.py:99-175
        accepts_fmha_config = False

        def support_cuda_graph(self) -> bool:
            return callable(getattr(self, "prepare_cuda_graph", None))

        @classmethod
        def support_parallelism_config(cls, parallelism_config) -> bool:
            return True


def _tokens_per_block(cfg) -> int:
    return int(getattr(cfg, "kernel_tokens_per_block", 0) or getattr(cfg, "tokens_per_block"))


@dataclass
class B200AttnParams:
    """== XQAParams (bindings/cuda/ops/CudaXqa.h:10-16): what prepare() hands to forward()."""
    kv_cache_offset: torch.Tensor          # [B,1,2,M] int32 page list
    sequence_lengths: torch.Tensor         # captured BY REFERENCE so graph replay can refresh it in place (xqa.py:78-80)
    batch_size: int
    max_seq_len: int
    workspace: torch.Tensor
    q_len: int = 1                         # query tokens per sequence (> 1: verification of speculative tokens)


_MAX_ROWS = 64       # query rows (group x q_len) per (sequence, kv head) of b200_paged_decode_attn(_multi)
_BEAM_MIN_UNITS = 128   # (request, kv head) pairs from which b200_paged_decode_attn_beam wins (measured, see beam_rows_fit)


def beam_rows_fit(head_num: int, kv_head_num: int, beam_width: int, requests: int) -> bool:
    """When a request's beams take the seat of one (sequence, kv head) in b200_paged_decode_attn_beam, which reads the K/V they
    share once: there is more than one beam, their group x beam_width query rows fit the kernel's row limit, and there are
    enough (request, kv head) pairs to fill the GPU with that many fewer, heavier CTAs. Everything else runs
    b200_paged_decode_attn on every beam.
    The boundary is measured (H100 80GB HBM3, 700 W; Hkv 8, D 128, ctx 2048, tools/kernel_bench.py attn-beam, beam / per row):
    256 pairs W 4 0.73; 128 pairs W 8 0.48 (group 4) and 0.72 (group 8); 64 pairs W 8 0.86, W 4 0.96, W 2 1.21; 32 pairs
    W 16 1.32 -- and at 64 pairs W 4 the whole step was 5 % slower with the beam kernel (tools/step_ab.py beam)."""
    group = head_num // max(kv_head_num, 1)
    return beam_width > 1 and group * beam_width <= _MAX_ROWS and requests * kv_head_num >= _BEAM_MIN_UNITS


def _q_len(attn_inputs) -> int:
    """Tokens per sequence of a decode step: max(input_lengths) when the inputs carry them (speculative verification,
    uniform across the batch), else 1."""
    lens = getattr(attn_inputs, "input_lengths", None)
    if lens is None or (torch.is_tensor(lens) and lens.numel() == 0):
        return 1
    return max(int(lens.max().item()) if torch.is_tensor(lens) else int(max(lens)), 1)


class B200DecodeAttnOp:
    def __init__(self, attn_configs):
        self.cfg = attn_configs

    def support(self, attn_inputs) -> bool:
        c = self.cfg
        if getattr(attn_inputs, "is_prefill", False):
            return False
        group = c.head_num // max(c.kv_head_num, 1)
        ok = (c.size_per_head in (64, 128, 256) and c.head_num % max(c.kv_head_num, 1) == 0
              and 1 <= group * _q_len(attn_inputs) <= _MAX_ROWS and _tokens_per_block(c) in (16, 32, 64, 128))
        kv_dtype = str(getattr(c, "kv_cache_dtype", "BASE"))
        return ok and "FP8" not in kv_dtype.upper() and torch.cuda.is_available() and \
            torch.cuda.get_device_capability() == (9, 0)

    def prepare(self, attn_inputs) -> B200AttnParams:
        block_ids = attn_inputs.kv_cache_kernel_block_id_device
        if block_ids is None:
            raise B200Error("decode should have kv cache block id.")          # XQAAttnOp.cc:66-67
        B = int(attn_inputs.sequence_lengths.shape[0])
        if block_ids.shape[0] != B:
            raise B200Error(f"kv blocks batch size expected [{B}] but got [{block_ids.shape[0]}]")
        page_list = ops.convert_block_table(block_ids)
        max_seq_len = int(getattr(self.cfg, "max_seq_len", 0)) or int(block_ids.shape[1]) * _tokens_per_block(self.cfg)
        # sequence_lengths may equal max_seq_len (tokens already cached): the kernel covers positions 0..sequence_lengths
        # inclusive, so the bound is max_seq_len + 1 exactly as XQAAttnOp.cc:147-149 passes it, capped by the page table
        q_len = _q_len(attn_inputs)
        max_seq_len = min(max_seq_len + q_len, int(block_ids.shape[1]) * _tokens_per_block(self.cfg))
        ws = ops.attn_workspace(B * q_len, self.cfg.head_num, self.cfg.kv_head_num, max_seq_len, block_ids.device)
        return B200AttnParams(page_list, attn_inputs.sequence_lengths, B, max_seq_len, ws, q_len)

    def update(self, params: B200AttnParams, attn_inputs) -> None:
        if params is None:
            raise B200Error("B200DecodeAttnOp::update received null params")
        self.update_kv_cache_offset(params.kv_cache_offset, attn_inputs.kv_cache_kernel_block_id_device)
        params.batch_size = int(attn_inputs.kv_cache_kernel_block_id_device.shape[0])
        params.sequence_lengths = attn_inputs.sequence_lengths

    def update_kv_cache_offset(self, kv_cache_offset: torch.Tensor, kv_cache_block_id_device: torch.Tensor) -> None:
        if kv_cache_offset.dim() != 4 or kv_cache_offset.shape[1] != 1 or kv_cache_offset.shape[2] != 2:
            raise B200Error("expects kv_cache_offset shape [batch, 1, 2, blocks]")          # XQAAttnOp.cc:31-32
        if kv_cache_offset.shape[0] != kv_cache_block_id_device.shape[0] or \
                kv_cache_offset.shape[3] != kv_cache_block_id_device.shape[1]:
            raise B200Error("shape mismatch: offset vs block table")
        ops.convert_block_table(kv_cache_block_id_device, out=kv_cache_offset)

    def forward(self, q: torch.Tensor, kv_cache, params: B200AttnParams) -> torch.Tensor:
        if kv_cache is None:
            raise B200Error("decode should have kv cache.")                                  # XQAAttnOp.cc:138
        base = kv_cache.kv_cache_base if hasattr(kv_cache, "kv_cache_base") else kv_cache
        seq = params.sequence_lengths
        if not seq.is_cuda and not seq.is_pinned():
            raise B200Error("sequence_lengths must be device-accessible (CUDA or pinned host memory)")
        q_scale = 1.0 / float(getattr(self.cfg, "q_scaling", 1.0) or 1.0)
        if params.q_len > 1:      # q [B*q_len, Hq*D] token-major -> [B, q_len, Hq, D]; out [B*q_len, Hq*D]
            D = base.shape[-1]
            q4 = q.reshape(params.batch_size, params.q_len, -1, D)
            out = ops.paged_decode_attn_multi(q4, base, params.kv_cache_offset, seq, params.max_seq_len, params.workspace,
                                              q_scale=q_scale)
            return out.reshape(params.batch_size * params.q_len, -1)
        return ops.paged_decode_attn(q, base, params.kv_cache_offset, seq, params.max_seq_len, params.workspace,
                                     q_scale=q_scale)


def _position_ids(attn_inputs) -> Optional[torch.Tensor]:
    """combo_position_ids of the inputs when present and non-empty: one rotation position per qkv row (entries <= 0 keep the
    cache slot)."""
    pid = getattr(attn_inputs, "combo_position_ids", None)
    return pid if torch.is_tensor(pid) and pid.numel() > 0 else None


class B200RopeKVCacheDecodeOp:
    """== FusedRopeKVCacheDecodeOp (rtp_llm/ops/fused_rope_kvcache_op.py:176-272): the rope config's style, rotary dim,
    scaling, Yarn / Llama3 factors, logn attention (attn_configs.use_logn_attn) and position ids, NeoX pairing; see rope.py
    for which kernel serves which config."""

    def __init__(self, attn_configs):
        self.cfg = attn_configs
        self.spec = rope.spec_of(getattr(attn_configs, "rope_config", None), int(attn_configs.size_per_head))
        self.use_logn_attn = bool(getattr(attn_configs, "use_logn_attn", False))

    def supported(self) -> bool:
        return rope.supported(self.spec, int(self.cfg.size_per_head))

    def prepare(self, attn_inputs):
        return attn_inputs

    def forward(self, qkv: torch.Tensor, kv_cache, page_list: torch.Tensor, sequence_lengths: torch.Tensor, q_len: int = 1,
                position_ids: Optional[torch.Tensor] = None):
        base = kv_cache.kv_cache_base if hasattr(kv_cache, "kv_cache_base") else kv_cache
        if position_ids is not None and (position_ids.device != qkv.device or position_ids.dtype != torch.int32):
            position_ids = position_ids.to(device=qkv.device, dtype=torch.int32)
        return rope.rope_append(self.spec, qkv, base, page_list, sequence_lengths, self.cfg.head_num, q_len=q_len,
                                use_logn_attn=self.use_logn_attn, position_ids=position_ids)


class B200DecodeImpl(FMHAImplBase):
    """Decode FMHA strategy; name contains no "XQA"/"TRT" so FMHAConfig toggles of other backends do not disable it
    (attn_factory.py:100-156)."""

    def __init__(self, attn_configs, attn_inputs, parallelism_config=None):
        self.need_rope_kv_cache = bool(getattr(attn_configs, "need_rope_kv_cache", True))
        self.fmha_impl = B200DecodeAttnOp(attn_configs)
        self.rope_kvcache_impl = B200RopeKVCacheDecodeOp(attn_configs)
        self.attn_inputs = attn_inputs
        self.fmha_params = self.fmha_impl.prepare(attn_inputs)
        self._captured_seq_lens = attn_inputs.sequence_lengths
        if self.need_rope_kv_cache:     # the cos/sin table is uploaded here, never inside a graph capture
            rope.table(self.rope_kvcache_impl.spec, attn_inputs.kv_cache_kernel_block_id_device.device)

    @staticmethod
    def support(attn_configs, attn_inputs) -> bool:
        """The attention shape is served, and so is the rope config when this impl applies it (an unserved rope style,
        non-NeoX pairing or an odd / oversized rotary dim falls through to another impl)."""
        if bool(getattr(attn_configs, "need_rope_kv_cache", True)) and not B200RopeKVCacheDecodeOp(attn_configs).supported():
            return False
        return B200DecodeAttnOp(attn_configs).support(attn_inputs)

    def forward(self, qkv: torch.Tensor, kv_cache, layer_idx: int = 0) -> torch.Tensor:
        """qkv [B*q_len, (Hq+2Hkv)*D], token-major (row b*q_len + j = token j of sequence b); q_len = 1 is plain decode."""
        q_len = self.fmha_params.q_len
        if q_len > 1 and qkv.shape[0] != self.fmha_params.batch_size * q_len:
            raise B200Error(f"qkv has {qkv.shape[0]} rows, expected batch {self.fmha_params.batch_size} x q_len {q_len}")
        if self.need_rope_kv_cache:
            q = self.rope_kvcache_impl.forward(qkv, kv_cache, self.fmha_params.kv_cache_offset,
                                               self.fmha_params.sequence_lengths, q_len, _position_ids(self.attn_inputs))
        else:
            q = qkv
        return self.fmha_impl.forward(q, kv_cache, self.fmha_params)

    def prepare_cuda_graph(self, attn_inputs) -> None:
        """Refresh per-step metadata IN PLACE (attention/common.py:88-138): page list, sequence lengths and position ids."""
        self.fmha_impl.update_kv_cache_offset(self.fmha_params.kv_cache_offset, attn_inputs.kv_cache_kernel_block_id_device)
        if attn_inputs.sequence_lengths is not self._captured_seq_lens:
            self._captured_seq_lens.copy_(attn_inputs.sequence_lengths, non_blocking=True)
        pid, captured = _position_ids(attn_inputs), _position_ids(self.attn_inputs)
        if pid is not None and captured is not None and pid is not captured:
            captured.copy_(pid, non_blocking=True)
