"""Synthetic AutoGPTQ act-order (desc_act) checkpoints for the act-order tests: qweight / qzeros / scales packed as in
tests/ckpt_util.py, plus the `.g_idx` tensor that maps each input row (in checkpoint order) to its quantisation group."""
import numpy as np
import torch

from tests.ckpt_util import _pack_cols, _pack_rows


def act_order_g_idx(rng, K, group):
    """AutoGPTQ desc_act: features visited in a random order `perm`, a new group every `group` of them; g_idx in the original
    row order: g_idx[k] = rank of k in perm // group."""
    perm = rng.permutation(K)
    rank = np.empty(K, np.int64)
    rank[perm] = np.arange(K)
    return (rank // group).astype(np.int32)


def make_act_order_layer(rng, K, N, g_idx, group=128, bits=4):
    """An AutoGPTQ act-order layer: qweight in the original row order, scales / qzeros row r = group r, and `.g_idx`. Returns
    (tensors, dense [K, N] = (q - z[g_idx[k]]) * s[g_idx[k]], q [K, N] unsigned, z, s)."""
    top = 1 << bits
    q = rng.integers(0, top, (K, N))
    z = rng.integers(1, top, (K // group, N))
    s = (np.abs(rng.standard_normal((K // group, N))) * (0.01 if bits == 4 else 6e-4) + (1e-3 if bits == 4 else 6e-5)).astype(np.float16)
    dense = (q - z[g_idx]).astype(np.float32) * s.astype(np.float32)[g_idx]
    t = dict(qweight=_pack_rows(q, bits), qzeros=_pack_cols(z - 1, list(range(8)), bits), scales=s, g_idx=np.array(g_idx, np.int32))
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in t.items()}, dense, q, z, s


def write_act_order_checkpoint(path, rng, hidden, heads, kv_heads, head_dim, inter, group=128, bits=4, trivial=False):
    """One act-order GPTQ decoder layer in HF naming: q / k / v share one g_idx and gate / up another (same input), o and
    down have their own. trivial=True stores g_idx[k] = k // group everywhere. Returns (names, dense, g_idx by input)."""
    from safetensors.torch import save_file
    shapes = dict(q=(hidden, heads * head_dim), k=(hidden, kv_heads * head_dim), v=(hidden, kv_heads * head_dim),
                  o=(heads * head_dim, hidden), gate=(hidden, inter), up=(hidden, inter), down=(inter, hidden))
    src = dict(q="qkv", k="qkv", v="qkv", o="o", gate="w13", up="w13", down="w2")
    gi = {}
    for key, (K, _) in shapes.items():
        if src[key] not in gi:
            gi[src[key]] = (np.arange(K) // group).astype(np.int32) if trivial else act_order_g_idx(rng, K, group)
    tensors, dense, names = {}, {}, {}
    for key, (K, N) in shapes.items():
        names[key] = f"model.layers.0.{key}"
        t, dense[key], *_ = make_act_order_layer(rng, K, N, gi[src[key]], group, bits)
        tensors.update({f"{names[key]}.{sfx}": v for sfx, v in t.items()})
    save_file(tensors, path)
    return names, dense, gi
