"""CPU tests of the host side of Qwen3 layers: the loader reads q_norm / k_norm gammas from a safetensors checkpoint (and names a
missing one), the C ABI, header and ctypes table carry the fused QK-norm + rope entries, and the Qwen3 configs."""
import os
import re

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, decode_step
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig
from tests import ckpt_util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("b200_qk_norm_rope_append", "b200_qk_norm_rope_append_ex")


def _qwen3_checkpoint(path, with_k_norm=True):
    """One Qwen3 layer in HF naming: the dense layer of ckpt_util plus self_attn.q_norm.weight / k_norm.weight [head_dim]."""
    from safetensors.torch import load_file, save_file
    rng = np.random.default_rng(3)
    D = 64
    names, _ = ckpt_util.write_checkpoint(path, rng, "none", 256, 4, 2, D, 256)
    tensors = load_file(path)
    norms = {"q_norm": torch.from_numpy((1 + 0.1 * rng.standard_normal(D)).astype(np.float32)).to(torch.bfloat16)}
    if with_k_norm:
        norms["k_norm"] = torch.from_numpy((1 + 0.1 * rng.standard_normal(D)).astype(np.float32)).to(torch.bfloat16)
    for k, v in norms.items():
        tensors[f"model.layers.0.self_attn.{k}.weight"] = v
    save_file(tensors, path)
    names.update(q_norm="model.layers.0.self_attn.q_norm", k_norm="model.layers.0.self_attn.k_norm")
    return names, norms


def test_loader_reads_the_qk_norm_gammas(tmp_path):
    path = str(tmp_path / "qwen3.safetensors")
    names, norms = _qwen3_checkpoint(path)
    ld = B200Loader(CheckpointReader(path), QuantConfig("none"), device="cpu", act_dtype=torch.float16)
    got = ld.qk_norms(names)
    assert sorted(got) == ["k_norm", "q_norm"]
    for k, v in got.items():
        assert v.dtype == torch.float16 and v.shape == (64,) and v.is_contiguous()
        assert torch.equal(v, norms[k].to(torch.float16))
    plain = {k: v for k, v in names.items() if k not in ("q_norm", "k_norm")}
    assert ld.qk_norms(plain) == {}                         # a layer without QK-norm loads none


def test_a_missing_norm_raises_the_readers_key_error(tmp_path):
    path = str(tmp_path / "qwen3.safetensors")
    names, _ = _qwen3_checkpoint(path, with_k_norm=False)
    ld = B200Loader(CheckpointReader(path), QuantConfig("none"), device="cpu")
    with pytest.raises(KeyError, match="k_norm.weight"):
        ld.qk_norms(names)
    with pytest.raises(KeyError, match="k_norm.weight"):   # before any weight is packed
        ld.layer(names, inter=256)


def test_fused_entries_are_declared_exported_and_typed():
    from rtp_llm_b200 import build
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200_decode_ops.h")).read(), flags=re.S)
    lib = _lib.load() if os.path.exists(build.LIB) else None
    for name in ENTRIES:
        assert re.search(rf"\bint {name}\(", hdr), name
        assert name in _lib.SIGNATURES
        if lib is not None:
            assert hasattr(lib, name)
    assert len(_lib.SIGNATURES["b200_qk_norm_rope_append"][1]) == 18
    assert len(_lib.SIGNATURES["b200_qk_norm_rope_append_ex"][1]) == 22


def test_argument_checks_reject_before_any_launch():
    lib = _lib.load()
    buf = torch.zeros(64, dtype=torch.int32)
    p = buf.data_ptr()
    assert lib.b200_qk_norm_rope_append(p, None, p, 1e-6, p, p, p, p, 0, 1, 1, 1, 128, 1, 16, 1e6, 1, None) != 0
    assert b"gamma" in lib.b200_last_error()
    assert lib.b200_qk_norm_rope_append(p, p, p, 1e-6, p, p, p, p, 0, 1, 1, 1, 96, 1, 16, 1e6, 1, None) != 0
    assert b"head_dim" in lib.b200_last_error()


def test_qwen3_configs():
    q8, q32, tiny = decode_step.QWEN3_8B, decode_step.QWEN3_32B, decode_step.TINY_QWEN3
    assert (q8.hidden, q8.layers, q8.head_num, q8.kv_head_num, q8.head_dim, q8.inter, q8.vocab) == (4096, 36, 32, 8, 128, 12288, 151936)
    assert (q32.hidden, q32.layers, q32.head_num, q32.kv_head_num, q32.inter) == (5120, 64, 64, 8, 25600)
    for c in (q8, q32, tiny):
        assert c.qk_norm and c.rope_base == 1e6 and c.eps == 1e-6
    assert q32.head_num * q32.head_dim != q32.hidden and tiny.head_num * tiny.head_dim != tiny.hidden
    for c in (decode_step.LLAMA3_8B, decode_step.LLAMA31_8B, decode_step.QWEN2_72B, decode_step.TINY):
        assert not c.qk_norm
