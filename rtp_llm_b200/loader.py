"""On-disk formats -> kernel layout: AutoGPTQ / AutoAWQ 4-bit group-wise checkpoints and plain FP16/BF16 weights for the
per-column INT8 path, read from safetensors and pushed through the device hooks exactly as the reference's loader does
(SURVEY 8 f-4).  What is mirrored, file:line in /root/reference:
  * tensor names   `<prefix>.qweight / .qzeros / .scales`                    model_loader/group_wise_quant_weight.py:32-36
  * which layers   qkv, o, w1 / w3 (merged into w13), w2                     group_wise_quant_weight.py:304-316;
                   Qwen3's q_norm / k_norm gammas `<prefix>.weight`, unquantised, when the layer names them
  * merge rules    q|k|v and gate|up concatenated along the OUTPUT axis (GPTQ qweight [K/8, N]: dim 1; AWQ qweight [K, N/8]: dim 1)
  * padding        the FFN inter size is padded to `align_size`: w2 along its INPUT rows (GPTQ qweight rows are packed 8:1 ->
                   align_size / 8; AWQ: align_size), zeros / scales by align_size / group_size rows; w1 / w3 along their
                   OUTPUT columns (group_wise_quant_weight.py:123-176, utils/model_weight.py:74-110 `pad`)
  * act-order      GPTQ `desc_act` checkpoints carry `<prefix>.g_idx`: rows are sorted by it (device.act_order_perm) and the
                   blob carries the order, except for w2, whose order is folded into w13's output columns (B200Loader.layer)
  * post-process   load_config.exported_device.preprocess_groupwise_weight_params(qweight, qzeros, scales, device, gptq, awq,
                   bits) (group_wise_quant_weight.py:392-425) -> here B200Impl (device.py); per-column INT8:
                   exported_device.apply_int8(kernel, device) (weight_only_quant_weight.py:94-105)
safetensors (the library) is plumbing for the file format, like torch is for device memory."""
from __future__ import annotations

import dataclasses
from typing import Dict, Optional

import torch

from . import ops
from .device import B200Impl, act_order_perm

QW, QZ, QS, GI = ".qweight", ".qzeros", ".scales", ".g_idx"


@dataclasses.dataclass
class QuantConfig:
    method: str              # "gptq" | "awq" | "int8" (per-column weight-only, quantised at load time) | "none"
    bits: int = 4
    group_size: int = 128    # 4-bit: 32, 64, 128 (or a larger multiple of 128), -1 = per channel; 8-bit: 128

    @property
    def gptq(self) -> bool:
        return self.method == "gptq"

    @property
    def awq(self) -> bool:
        return self.method == "awq"


def pad_dim(t: torch.Tensor, align: int, dim: int, value: int = 0) -> torch.Tensor:
    """utils/model_weight.py:74-110: zero-pad `dim` up to a multiple of `align` (0 = no padding)."""
    if align <= 0:
        return t.contiguous()
    size = t.shape[dim]
    extra = (-size) % align
    if extra == 0:
        return t.contiguous()
    shape = list(t.shape)
    shape[dim] = extra
    return torch.cat([t, torch.full(shape, value, dtype=t.dtype, device=t.device)], dim=dim).contiguous()


class CheckpointReader:
    """Lazy view of one or more .safetensors files (AutoGPTQ / AutoAWQ / HF layout)."""

    def __init__(self, *paths: str):
        from safetensors import safe_open
        self._files = [safe_open(p, framework="pt", device="cpu") for p in paths]
        self._where = {k: f for f in self._files for k in f.keys()}

    def __contains__(self, name: str) -> bool:
        return name in self._where

    def get(self, name: str) -> torch.Tensor:
        if name not in self._where:
            raise KeyError(f"tensor {name!r} not found in the checkpoint")
        return self._where[name].get_tensor(name)


class B200Loader:
    """Builds the weights of one decoder layer in the kernel's layout. `names` maps the reference's logical weights to
    checkpoint prefixes, e.g. dict(q="model.layers.0.self_attn.q_proj", k=..., v=..., o=..., gate=..., up=..., down=...)."""

    def __init__(self, reader: CheckpointReader, quant: QuantConfig, device="cuda", act_dtype=torch.float16, align_size: int = 0,
                 fuse_silu: bool = True):
        self.r, self.q, self.device, self.act_dtype, self.align, self.fuse_silu = reader, quant, torch.device(device), act_dtype, align_size, fuse_silu
        self.impl = B200Impl(device, act_dtype)

    # ---- group-wise INT4 / INT8 (GPTQ / AWQ)
    def _triple(self, prefix: str):
        return self.r.get(prefix + QW), self.r.get(prefix + QZ), self.r.get(prefix + QS)

    def groupwise_tensors(self, prefixes, pad_in: int = 0, pad_out: int = 0):
        """Merge + pad + unpack on the host: the loader's UN-permuted tensors (q_packed uint8 [K, N/2] two's-complement
        nibbles, zeros_x_scales fp16 [K/g, N], scales fp16 [K/g, N]) -- what preprocess_groupwise_weight_params computes before
        its device-specific re-layout (device_impl.py:242-300)."""
        q = self.q
        if q.bits not in (4, 8):
            raise ValueError(f"group-wise checkpoints: bits must be 4 or 8, got {q.bits}")
        pad_div = 32 // q.bits                                        # group_wise_quant_weight.py:130
        qws, qzs, qss = zip(*[self._triple(p) for p in prefixes])
        if pad_out:                                                   # w1 / w3: the inter size is their OUTPUT axis
            qws = [pad_dim(w, pad_out if q.gptq else pad_out // pad_div, 1) for w in qws]
            qzs = [pad_dim(z, pad_out // pad_div, 1) for z in qzs]
            qss = [pad_dim(s, pad_out, 1) for s in qss]
        qw, qz, qs = torch.cat(qws, dim=1), torch.cat(qzs, dim=1), torch.cat(qss, dim=1)
        if pad_in:                                                    # w2: the inter size is its INPUT axis
            qw = pad_dim(qw, pad_in // pad_div if q.gptq else pad_in, 0)
            # per channel (group_size -1): the one row of zeros / scales covers the padded rows too
            rows = max(pad_in // q.group_size, 1) if q.group_size > 0 else 0
            qz = pad_dim(qz, rows, 0)
            qs = pad_dim(qs, rows, 0)
        return self.impl.unpack_groupwise(qw, qz, qs.to(torch.float16), q.gptq, q.awq, q.bits)

    def act_order(self, prefixes) -> Optional[torch.Tensor]:
        """The row order (act_order_perm) the merged weights `prefixes` share, or None (no act-order: AWQ, no `.g_idx`, or a
        trivial one). Merged parts see the same input, so AutoGPTQ gives them the same g_idx; different ones cannot be served by
        one sorted weight and raise ValueError."""
        if not self.q.gptq:
            return None
        perms = []
        for p in prefixes:
            K = self.r.get(p + QW).shape[0] * 32 // self.q.bits      # GPTQ qweight: [K * bits / 32, N]
            perms.append(act_order_perm(self.r.get(p + GI), self.q.group_size, K) if p + GI in self.r else None)
        for p, perm in zip(prefixes[1:], perms[1:]):
            same = (perm is None and perms[0] is None) or (perm is not None and perms[0] is not None and torch.equal(perm, perms[0]))
            if not same:
                raise ValueError(f"act-order: {prefixes[0]} and {p} are merged into one weight but have different g_idx")
        return perms[0]

    def sorted_tensors(self, prefixes, pad_in: int = 0, pad_out: int = 0, col_perm: Optional[torch.Tensor] = None):
        """groupwise_tensors with act-order applied on the host: (q, zeros_x_scales, scales, perm). Rows sorted by g_idx (sorted
        row j = checkpoint row perm[j]; perm None without act-order). col_perm: w2's order, applied to each half of a gate|up
        weight's output columns (the fold, see layer())."""
        q_packed, zs, scales = self.groupwise_tensors(prefixes, pad_in, pad_out)
        perm = self.act_order(prefixes)
        if perm is not None:
            # w2 padding: the padded rows are groups of their own and keep their place after the sorted rows
            perm = torch.cat([perm, torch.arange(perm.numel(), q_packed.shape[0])])
            q_packed = q_packed[perm]
        if col_perm is not None:
            half = scales.shape[1] // 2
            cp = torch.cat([col_perm, torch.arange(col_perm.numel(), half)])             # the padded inter columns stay put
            order = torch.cat([cp, cp + half])
            q_packed = ops.permute_columns(q_packed, order, packed_int4=self.q.bits == 4)
            zs, scales = ops.permute_columns(zs, order), ops.permute_columns(scales, order)
        return q_packed, zs, scales, perm

    def _groupwise(self, prefixes, pad_in: int = 0, pad_out: int = 0, gate_up_inter: int = 0,
                   col_perm: Optional[torch.Tensor] = None, keep_perm: bool = True) -> ops.PackedWeight:
        """keep_perm=False: the weight's own row order is folded into another weight (w2 into w13), so the blob omits it."""
        q_packed, zs, scales, perm = self.sorted_tensors(prefixes, pad_in, pad_out, col_perm)
        q_packed, zs, scales = q_packed.to(self.device), zs.to(self.act_dtype).to(self.device), scales.to(self.act_dtype).to(self.device)
        if gate_up_inter:
            q_packed = ops.interleave_gate_up(q_packed, gate_up_inter, packed_int4=self.q.bits == 4)
            zs, scales = ops.interleave_gate_up(zs, gate_up_inter), ops.interleave_gate_up(scales, gate_up_inter)
        pack = ops.pack_w4 if self.q.bits == 4 else ops.pack_w8g     # 8-bit: q_s int8 [K, N], one byte per weight
        return pack(q_packed.contiguous(), scales.contiguous(), zs.contiguous(), self.q.group_size,
                    perm=perm if keep_perm else None)

    # ---- per-column INT8 (quantised at load time from FP16/BF16 weights) and plain FP16
    def _dense(self, prefixes, pad_in: int = 0, pad_out: int = 0, gate_up_inter: int = 0) -> ops.PackedWeight:
        ws = [self.r.get(p + ".weight").t().contiguous() for p in prefixes]          # HF stores [N, K]; the reference works on [K, N]
        if pad_out:
            ws = [pad_dim(w, pad_out, 1) for w in ws]
        w = torch.cat(ws, dim=1)
        if pad_in:
            w = pad_dim(w, pad_in, 0)
        if self.q.method == "int8":
            qv, scale = self.impl.symmetric_quantize_last_axis_of_batched_matrix(w.float())
            qv, scale = qv.to(self.device), scale.to(self.act_dtype).to(self.device)
            if gate_up_inter:
                qv, scale = ops.interleave_gate_up(qv, gate_up_inter), ops.interleave_gate_up(scale, gate_up_inter)
            return ops.pack_w8(qv.contiguous(), scale.contiguous())
        w = w.to(self.act_dtype).to(self.device)
        if gate_up_inter:
            w = ops.interleave_gate_up(w, gate_up_inter)
        return ops.pack_f16(w)

    def _load(self, prefixes, **kw) -> ops.PackedWeight:
        return self._groupwise(prefixes, **kw) if self.q.method in ("gptq", "awq") else self._dense(prefixes, **kw)

    def qk_norms(self, names: Dict[str, str]) -> Dict[str, torch.Tensor]:
        """Qwen3's QK-norm gammas: `<names["q_norm"]>.weight` / `<names["k_norm"]>.weight` (HF: ...self_attn.q_norm.weight) as
        contiguous act-dtype [head_dim] tensors on the loader's device, for the names given. A missing tensor raises the
        reader's KeyError, which names it."""
        return {k: self.r.get(names[k] + ".weight").to(self.act_dtype).to(self.device).contiguous()
                for k in ("q_norm", "k_norm") if k in names}

    def layer(self, names: Dict[str, str], inter: Optional[int] = None) -> Dict[str, ops.PackedWeight]:
        """qkv / o / w13 / w2 of one decoder layer, and q_norm / k_norm (qk_norms) when `names` has them. `inter` = the
        checkpoint's FFN inter size (needed for padding + fusion).

        Act-order: qkv, o and w13 carry their row order (the GEMM gathers x). w2's order P2 is folded into w13 instead: column i
        of w2's input is SiLU(gate_i) * up_i, so w13 with its gate and up columns permuted by P2 emits act[:, P2] directly and
        the sorted w2 needs no gather."""
        norms = self.qk_norms(names)      # first: a missing norm fails before any weight is packed
        out = {"qkv": self._load([names["q"], names["k"], names["v"]]), "o": self._load([names["o"]]), **norms}
        pad = self.align
        inter_p = inter if inter is None or not pad else (inter + pad - 1) // pad * pad
        fuse = self.fuse_silu and inter_p is not None and inter_p % 64 == 0
        w13_kw = dict(pad_out=pad, gate_up_inter=inter_p if fuse else 0)
        if self.q.method in ("gptq", "awq"):
            p2 = self.act_order([names["down"]])
            out["w13"] = self._groupwise([names["gate"], names["up"]], col_perm=p2, **w13_kw)
            out["w2"] = self._groupwise([names["down"]], pad_in=pad, keep_perm=False)
        else:
            out["w13"] = self._dense([names["gate"], names["up"]], **w13_kw)
            out["w2"] = self._dense([names["down"]], pad_in=pad)
        out["w13_fused_silu"] = fuse
        return out
