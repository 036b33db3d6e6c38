"""Host-side mirror of the loader's device hooks: DeviceBase.{apply_int8, preprocess_groupwise_weight_params,
preprocess_weights_for_mixed_gemm} (/root/reference/rtp_llm/device/device_base.py:56-90), instance stored in
LoadConfig.exported_device (model_loader/loader.py:79).

The unpack / quantise arithmetic restates device_impl.py:148-300 in torch (bit-exact against the reference's code on the
golden fixtures, tests/test_host_logic.py); only the final re-layout differs: instead of the FT sm80 interleave
(device_impl.py:392-479) weights go into the TMA-friendly blobs of include/b200_decode_ops.h."""
from __future__ import annotations

import torch

from . import ops


def unpack_int32_into_int16(w_packed: torch.Tensor, int8: bool = False) -> torch.Tensor:
    """device_impl.py:147-161: int32 words -> bytes (8-bit checkpoints) or nibbles (low nibble first) along the last axis."""
    b = w_packed.contiguous().view(torch.uint8)
    if int8:
        return b.to(torch.int16)
    out = torch.empty(b.shape[0], b.shape[1] * 2, dtype=torch.int16, device=b.device)
    out[:, ::2] = (b % 16).to(torch.int16)
    out[:, 1::2] = (b // 16).to(torch.int16)
    return out


def reverse_awq_order(t: torch.Tensor) -> torch.Tensor:
    """device_impl.py:163-171."""
    return t.reshape(-1, 2, 4).transpose(2, 1).reshape(t.shape)


def pack_int8_tensor_to_packed_int4(t: torch.Tensor) -> torch.Tensor:
    """device_impl.py:204-209: two's-complement nibbles, low nibble = even column."""
    u = (t.to(torch.int16) & 0xF).to(torch.uint8)
    return (u[:, 1::2] * 16 + u[:, ::2]).contiguous()


def act_order_perm(g_idx, group: int, K: int):
    """Row order of a GPTQ act-order (desc_act) weight: `perm` int64 [K] with sorted row j = checkpoint row perm[j] (a stable
    argsort of g_idx), so that group r becomes rows [r*group, (r+1)*group) and the usual blob formats serve the weight; the
    GEMM then consumes x[:, perm]. None when g_idx is absent or trivial (g_idx[k] == k // group: static groups, no act-order,
    per channel), so those weights take the unpermuted path bit for bit. group -1 means per channel (group = K).

    AutoGPTQ stores g_idx in the checkpoint's row order, g_idx[k] = (rank of k in the act-order) // group, so every group has
    exactly `group` rows; anything else is not a checkpoint this layout can serve and raises ValueError."""
    if g_idx is None:
        return None
    if group == -1:
        group = K
    g = torch.as_tensor(g_idx).detach().to("cpu", torch.int64).reshape(-1)
    if group <= 0 or K % group:
        raise ValueError(f"g_idx: group size {group} does not divide K={K}")
    if g.numel() != K:
        raise ValueError(f"g_idx has {g.numel()} entries, expected K={K}")
    groups = K // group
    if g.numel() and (int(g.min()) < 0 or int(g.max()) >= groups):
        raise ValueError(f"g_idx values must lie in [0, {groups}) (K={K}, group {group}), got [{int(g.min())}, {int(g.max())}]")
    counts = torch.bincount(g, minlength=groups)
    if not bool((counts == group).all()):
        r = int(torch.nonzero(counts != group)[0])
        raise ValueError(f"g_idx: group {r} has {int(counts[r])} rows, every group must have exactly {group}")
    if torch.equal(g, torch.arange(K) // group):
        return None
    return torch.sort(g, stable=True).indices


class B200Impl:
    """Drop-in for CudaImpl's weight hooks. The returned `kernel` tensors are self-describing blobs (ops.PackedWeight: a
    trailer inside the tensor names format / K / N), so they survive the loader's `.contiguous().to(device)`, clones and
    state-dict round trips; B200WeightOnlyLinear rebuilds the description with PackedWeight.from_tensor()."""

    def __init__(self, device="cuda", act_dtype=torch.float16):
        self.device, self.act_dtype = torch.device(device), act_dtype

    # -- device_impl.py:183-202 / 215-222
    def symmetric_quantize_last_axis_of_batched_matrix(self, weight: torch.Tensor, quant_mode=torch.int8):
        amax = torch.clamp(weight.abs().max(dim=0)[0], min=1e-8)
        scale = amax / 128.0
        q = torch.clamp((weight / scale).round(), -128, 127).char()
        return q, scale

    def apply_int8(self, tensor: torch.Tensor, device: str = "cuda"):
        shape = tensor.shape
        q, scale = self.symmetric_quantize_last_axis_of_batched_matrix(tensor.reshape(shape[0], -1).float())
        packed = ops.pack_w8(q.to(self.device).contiguous(), scale.to(self.act_dtype).to(self.device))
        return packed.data, scale.to(self.device)

    # -- device_impl.py:242-300
    def unpack_groupwise(self, qweight_int32, qzeros_int32, scales_fp16, gptq: bool, awq: bool, weight_bits: int = 4):
        """Returns the loader's UN-permuted tensors: 4-bit (q_packed uint8 [K,N/2], zeros_x_scales fp16, scales fp16);
        8-bit (device_impl.py:256-258: zero shift 128, no nibble packing) (q_s int8 [K,N], zeros_x_scales, scales)."""
        if weight_bits not in (4, 8):
            raise ValueError(f"group-wise weight_bits must be 4 or 8, got {weight_bits}")
        is_int8 = weight_bits == 8
        shift = 128 if is_int8 else 8
        qweight = qweight_int32.reshape(qweight_int32.shape[0], -1)
        qzeros = qzeros_int32.reshape(qzeros_int32.shape[0], -1)
        scales = scales_fp16.reshape(scales_fp16.shape[0], -1)
        if awq:
            q = reverse_awq_order(unpack_int32_into_int16(qweight, is_int8) - shift)
        elif gptq:
            q = (unpack_int32_into_int16(qweight.T.contiguous(), is_int8).T.contiguous() - shift)
        else:
            raise ValueError("need gptq or awq")
        q = q.to(torch.int8)
        q_out = q.contiguous() if is_int8 else pack_int8_tensor_to_packed_int4(q)
        z = unpack_int32_into_int16(qzeros, is_int8)
        if awq:
            z = reverse_awq_order(z)
        zeros_x_scales = ((-z + shift - (1 if gptq else 0)) * scales).half()
        return q_out, zeros_x_scales, scales

    def preprocess_groupwise_weight_params(self, qweight_int32, qzeros_int32, scales_fp16, device: str, gptq: bool,
                                           awq: bool, weight_bits: int, g_idx=None):
        """g_idx: a GPTQ checkpoint's `.g_idx` (act-order). The rows are sorted by it and the blob carries the order
        (act_order_perm); None or a trivial g_idx gives the plain blob."""
        q_packed, zs, scales = self.unpack_groupwise(qweight_int32, qzeros_int32, scales_fp16, gptq, awq, weight_bits)
        perm = None
        if g_idx is not None:
            K, rows = q_packed.shape[0], scales.reshape(scales.shape[0], -1).shape[0]
            perm = act_order_perm(g_idx, K // rows if rows and K % rows == 0 else 0, K)
            if perm is not None:
                q_packed = q_packed[perm.to(q_packed.device)]
        kernel = self.preprocess_weights_for_mixed_gemm(q_packed, torch.int8 if weight_bits == 8 else torch.quint4x2, scales=scales,
                                                        zeros_x_scales=zs, perm=perm)
        return kernel, zs.to(self.device), scales.to(self.device)

    # -- replaces device_impl.py:392-479
    def preprocess_weights_for_mixed_gemm(self, tensor: torch.Tensor, quant_mode, arch: str = "", scales=None,
                                          zeros_x_scales=None, perm=None):
        if quant_mode == torch.int8 and zeros_x_scales is None:
            raise ValueError("INT8 per-column weights are packed by apply_int8 (the scale rides along)")
        assert scales is not None and zeros_x_scales is not None, "the b200 group-wise blobs carry scales and zero*scale"
        # the reference's hook takes no group argument: the group is what the scales' row count implies
        K, N = tensor.shape[0], tensor.shape[1] * (1 if quant_mode == torch.int8 else 2)
        rows = scales.numel() // N
        group = K // rows if rows and K % rows == 0 else 0
        scales, zeros_x_scales = scales.reshape(rows, N), zeros_x_scales.reshape(rows, N)
        if quant_mode == torch.int8:        # 8-bit group-wise
            if group != 128:
                raise ValueError(f"8-bit group-wise weights: group size {group or f'K/{rows}'} unsupported (128 only; K={K}, "
                                 f"{rows} scale rows)")
            return ops.pack_w8g(tensor.to(self.device).contiguous(), scales.to(self.act_dtype).to(self.device).contiguous(),
                                zeros_x_scales.to(self.act_dtype).to(self.device).contiguous(), perm=perm).data
        if group not in (32, 64) and (group < 128 or group % 128):
            raise ValueError(f"INT4 group-wise weights: group size {group or f'K/{rows}'} unsupported (32, 64 or a multiple of "
                             f"128, per-channel included; K={K}, {rows} scale rows)")
        packed = ops.pack_w4(tensor.to(self.device).contiguous(), scales.to(self.act_dtype).to(self.device).contiguous(),
                             zeros_x_scales.to(self.act_dtype).to(self.device).contiguous(), group, perm=perm)
        return packed.data
