"""Host-side mirror of the reference's Linear seam: a LinearBase strategy for weight-only INT4 (GPTQ/AWQ g128 / g64 / g32) / INT8 /
FP16 weights (/root/reference/rtp_llm/models_py/modules/factory/linear/linear_base.py:16-102; registration
factory.py:43-51; the CUDA strategies that exist today, impl/cuda/__init__.py:15-28, do not cover weight-only INT4/INT8 --
an int8-typed weight with scales raises "No suitable Linear strategy", factory.py:113-120).

Weights arrive as the loader produced them: for quantised layers `weight` is the output of
B200Impl.preprocess_weights_for_mixed_gemm (already in the kernel's blob layout, see device.py), `weight_scales` the scales;
zeros*scales are stashed inside the INT4 blob at load time, which is why this strategy does not need the `W.*_z` tensors the
reference's call sites do not pass (SURVEY 8b)."""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from . import ops
from ._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8, B200Error

try:
    from rtp_llm.models_py.modules.factory.linear.linear_base import LinearBase  # type: ignore
except Exception:  # noqa: BLE001
    class LinearBase(nn.Module):  # same surface as linear_base.py:16-102
        def __init__(self, *a, **k):
            super().__init__()

        def maybe_cache_quant_scale(self, max_len: int) -> None:
            pass

def _workspace(device, max_batch, K, N):
    """Scratch of ONE linear module (split-K partials + semaphores), sized once at construction for its own (K, N) and the
    largest batch a call handles: never reallocated, never shared -- safe under CUDA-graph capture and with several streams
    (a process-wide buffer that grows on demand would leave captured graphs pointing at freed memory and let two GEMMs on
    different streams share semaphores)."""
    need = int(ops._lib.load().b200_wo_gemm_workspace_bytes(max_batch, N, K))
    return torch.zeros(max(need, 16384), dtype=torch.uint8, device=device)


def _quant_method(quant_config) -> str:
    if quant_config is None:
        return ""
    for attr in ("get_method", "method", "quant_method", "name"):
        v = getattr(quant_config, attr, None)
        if callable(v):
            v = v()
        if v:
            return str(v).lower()
    return type(quant_config).__name__.lower()


class B200WeightOnlyLinear(LinearBase):
    MAX_BATCH = 128

    @classmethod
    def can_handle(cls, quant_config, weight, weight_scales, hw_kernel_config=None, weight_scale_2=None,
                   input_scale=None) -> bool:
        if weight_scale_2 is not None or input_scale is not None:
            return False
        if weight_scales is None:
            return weight.dtype in (torch.float16, torch.bfloat16)
        m = _quant_method(quant_config)
        return weight.dtype in (torch.int8, torch.uint8) and any(k in m for k in ("int8", "awq", "gptq", "weightonly", "w4a16"))

    def __init__(self, weight, weight_scales=None, input_scales=None, bias=None, quant_config=None, weight_scale_2=None):
        super().__init__(weight, weight_scales, input_scales, bias, quant_config, weight_scale_2)
        self.bias = bias
        if weight_scales is None:                       # FP16/BF16: reference stores [K, N]
            self.packed = ops.pack_f16(weight)
        elif isinstance(weight, ops.PackedWeight):
            self.packed = weight
        else:                                           # tensor produced by B200Impl.preprocess_* (device.py), or any copy of it
            self.packed = ops.PackedWeight.from_tensor(weight)
        if self.packed.fmt == B200_FMT_INT8 and self.packed.col_scale is None:
            self.packed.col_scale = weight_scales
        self._ws = _workspace(self.packed.data.device, self.MAX_BATCH, self.packed.K, self.packed.N)
        # act-order weights: x[:, perm] is gathered here before the GEMM; 16-bit activations of either dtype (viewed at call
        # time), sized once like the workspace so that captured graphs keep pointing at it
        self._x_perm = (torch.empty(self.MAX_BATCH * self.packed.K * 2, dtype=torch.uint8, device=self.packed.data.device)
                        if self.packed.perm is not None else None)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        lead = input.shape[:-1]
        x = input.reshape(-1, input.shape[-1])
        if x.shape[0] == 0:                              # as F.linear: an empty [*lead, N], no launch
            return input.new_empty((*lead, self.packed.N))
        if not x.is_contiguous():
            x = x.contiguous()
        if self.packed.col_scale is not None and self.packed.col_scale.dtype != x.dtype:
            self.packed.col_scale = self.packed.col_scale.to(x.dtype).contiguous()   # the loader keeps INT8 scales in fp32 (device_impl.py:190)
        ws = self._ws
        xp = None if self._x_perm is None else self._x_perm.view(x.dtype).view(self.MAX_BATCH, self.packed.K)
        outs = []
        for i in range(0, x.shape[0], self.MAX_BATCH):   # decode batches are <= 128; larger inputs go in slabs
            outs.append(ops.wo_gemm(x[i:i + self.MAX_BATCH], self.packed, ws, bias=self.bias, x_perm=xp))
        y = outs[0] if len(outs) == 1 else torch.cat(outs, 0)
        return y.reshape(*lead, self.packed.N)
