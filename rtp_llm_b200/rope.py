"""The rope config of the attention seams: which decode rope kernel serves it, and the cos/sin table the reference's decode op
reads for Base and Yarn.

A rope config is duck-typed on the reference's RopeConfig field names (cpp/model_utils/RopeConfig.h:21-42): style, dim, base,
scale, factor1, factor2, max_pos, extrapolation_factor, mscale, is_neox_style; absent fields take the defaults below (an
absent style is Base, an absent or zero dim is the head size). The table is built on the host with the torch calls of
RopeCache.cc:16-85 (genBaseCache / genYarnCache), laid out as getRopeCache(interleave = true) lays it out -- fp32
[int(max_pos * scale)][dim] of (cos, sin) pairs -- and uploaded once per config and device. For Yarn the table and the
in-kernel formula disagree (DESIGN.md §4); the decode op reads the table whenever it exists, so the table is what is served.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from . import _lib

# RopeStyle (RopeConfig.h:7-16)
NO, BASE, GLM2, DYNAMIC_NTK, QWEN_DYNAMIC_NTK, YARN, LLAMA3, MROPE = range(8)
SERVED_STYLES = (NO, BASE, DYNAMIC_NTK, QWEN_DYNAMIC_NTK, YARN, LLAMA3)   # Glm2 and 3-D Mrope positions are not built
TABLE_STYLES = (BASE, YARN)                                                # RopeCache.cc builds a table for these two


@dataclass(frozen=True)
class RopeSpec:
    style: int = BASE
    dim: int = 0
    base: float = 10000.0
    scale: float = 1.0
    factor1: float = 0.0
    factor2: float = 0.0
    max_pos: int = 0
    extrapolation_factor: float = 1.0
    mscale: float = 1.0
    is_neox_style: bool = True


def spec_of(rope_config, head_dim: int) -> RopeSpec:
    """The fields of a rope config object (None: plain Base at base 10000), with dim 0 resolved to head_dim."""
    d = RopeSpec()
    if rope_config is None:
        return RopeSpec(dim=head_dim)

    def get(name, cast):
        v = getattr(rope_config, name, None)
        return getattr(d, name) if v is None else cast(v)
    return RopeSpec(style=get("style", int), dim=get("dim", int) or head_dim, base=get("base", float), scale=get("scale", float),
                    factor1=get("factor1", float), factor2=get("factor2", float), max_pos=get("max_pos", int),
                    extrapolation_factor=get("extrapolation_factor", float), mscale=get("mscale", float),
                    is_neox_style=get("is_neox_style", bool))


def supported(spec: RopeSpec, head_dim: int) -> bool:
    """True when b200_rope_append(_ex)(_multi) computes this config's rotation: a served style, NeoX pairing, an even rotary
    dim no larger than the head."""
    return (spec.style in SERVED_STYLES and spec.is_neox_style and spec.dim % 2 == 0 and 0 < spec.dim <= head_dim
            and (spec.style == NO or spec.base > 1.0))


def is_plain_base(spec: RopeSpec, head_dim: int) -> bool:
    """Base rotation over the whole head at scale 1: what b200_rope_append computes (given no logn and no position ids)."""
    return spec.style == BASE and spec.scale == 1.0 and spec.dim == head_dim and spec.is_neox_style


def c_config(spec: RopeSpec) -> _lib.RopeConfig:
    return _lib.RopeConfig(style=spec.style, dim=spec.dim, base=spec.base, scale=spec.scale, factor1=spec.factor1,
                           factor2=spec.factor2, max_pos=spec.max_pos, extrapolation_factor=spec.extrapolation_factor,
                           mscale=spec.mscale)


def build_table(spec: RopeSpec) -> Optional[torch.Tensor]:
    """CPU fp32 [int(max_pos * scale), dim] interleaved (cos, sin) table for Base and Yarn (None for other styles, or when
    the config covers no position). Positions past the table are computed in the kernel, as in the reference."""
    positions = int(spec.max_pos * spec.scale)
    if spec.style not in TABLE_STYLES or positions <= 0:
        return None
    dim, theta, scale = spec.dim, spec.base, spec.scale
    if spec.style == BASE:                                                       # RopeCache.cc:16-44
        inv_freq = 1.0 / torch.pow(torch.tensor(float(theta)), torch.arange(0, dim, 2).float() / dim)
        t = torch.arange(positions).float()
        t.div_(scale)
        freqs = torch.outer(t, inv_freq)
        cos, sin = freqs.cos(), freqs.sin()
    else:                                                                        # RopeCache.cc:46-85
        pos_freqs = torch.pow(torch.tensor(float(theta)), torch.arange(0, dim, 2).float() / dim)
        inv_e, inv_i = 1.0 / pos_freqs, 1.0 / (scale * pos_freqs)
        corr = lambda nrot: float(dim * math.log(spec.max_pos / (nrot * 2.0 * math.pi))) / (2.0 * math.log(theta))
        low = float(max(0, int(math.floor(corr(spec.factor1)))))
        high = float(min(dim - 1, int(math.ceil(corr(spec.factor2)))))
        if abs(low - high) < 1e-6:
            high += 0.001
        ramp = torch.clamp((torch.arange(dim // 2).float() - low) / (high - low), 0, 1)
        mask = (1.0 - ramp) * spec.extrapolation_factor
        inv_freq = inv_i * (1.0 - mask) + inv_e * mask
        freqs = torch.outer(torch.arange(positions).float(), inv_freq)
        cos, sin = freqs.cos() * spec.mscale, freqs.sin() * spec.mscale
    return torch.stack([cos, sin], dim=-1).reshape(positions, -1).contiguous()


_TABLES: Dict[Tuple[RopeSpec, str], Optional[torch.Tensor]] = {}


def table(spec: RopeSpec, device) -> Optional[torch.Tensor]:
    """build_table(spec) on `device`, built and uploaded once per (config, device)."""
    key = (spec, str(torch.device(device)))
    if key not in _TABLES:
        t = build_table(spec)
        _TABLES[key] = None if t is None else t.to(device)
    return _TABLES[key]


def rope_append(spec: RopeSpec, qkv, kv_cache_base, page_list, sequence_lengths, head_num: int, q_out=None, q_len: int = 1,
                use_logn_attn: bool = False, position_ids=None, qk_norm=None):
    """Rotate q and k of qkv [B*q_len, (Hq+2Hkv)*D] and append K/V for any served config. A plain Base config without logn
    and position ids runs b200_rope_append(_multi) -- the bits callers that only set `base` have always had -- and every other
    config runs b200_rope_append_ex(_multi), with the cos/sin table for Base and Yarn.
    qk_norm = (q_gamma, k_gamma, eps): Qwen3's QK-RMSNorm of each q and k head first, in the same launch
    (b200_qk_norm_rope_append(_ex), picked by the same rule); qkv is then only read."""
    from . import ops
    D = kv_cache_base.shape[-1]
    if is_plain_base(spec, D) and not use_logn_attn and position_ids is None:
        if qk_norm is not None:
            return ops.qk_norm_rope_append(qkv, *qk_norm, kv_cache_base, page_list, sequence_lengths, head_num, spec.base,
                                           q_out=q_out, q_len=q_len)
        return ops.rope_append(qkv, kv_cache_base, page_list, sequence_lengths, head_num, spec.base, q_out=q_out, q_len=q_len)
    ex = dict(q_out=q_out, position_ids=position_ids, cos_sin_cache=table(spec, qkv.device), use_logn_attn=use_logn_attn,
              q_len=q_len)
    if qk_norm is not None:
        return ops.qk_norm_rope_append_ex(qkv, *qk_norm, kv_cache_base, page_list, sequence_lengths, head_num, c_config(spec), **ex)
    return ops.rope_append_ex(qkv, kv_cache_base, page_list, sequence_lengths, head_num, c_config(spec), **ex)
