"""INT4 group 64 / 32 / per-channel on the host (no GPU): blob sizes and argument checks of the C ABI, the group -> blob format
mapping of ops.w4_format, and AutoGPTQ / AutoAWQ checkpoints at those groups through B200Loader.groupwise_tensors, checked
against the dense weight the checkpoint means. The kernel side is tests/test_gpu_w4_groups.py."""
import ctypes

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200.device import B200Impl
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig
from tests import ckpt_util


def test_packed_bytes_of_the_group_formats():
    lib = _lib.load()
    # 8192 nibble bytes + 512 bytes of {scale, zero*scale} per group of the (128 x 128) block
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4_G64, 256, 256) == 2 * 2 * 9216
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4_G32, 256, 256) == 2 * 2 * 10240
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4_G32, 384, 200) == 3 * 2 * 10240     # N padded to 128-feature tiles
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4_G64, 100, 256) == 0               # K not a multiple of 128
    assert 9216 % 512 == 0 and 10240 % 512 == 0                                              # barriers after the ring stay aligned
    for unknown in (7, 9):
        assert lib.b200_wo_gemm_packed_bytes(unknown, 256, 256) == 0


def test_pack_w4_and_wo_gemm_rs_argument_checks():
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    regs = (ctypes.c_void_p * 8)(*([p.value] * 8))
    for group in (48, 256, 0, -1):
        assert lib.b200_pack_w4(p, p, p, 256, 256, group, p, None) == -1 and b"group" in lib.b200_last_error()
    assert lib.b200_pack_w4(p, p, p, 100, 256, 64, p, None) == -1 and b"multiple of 128" in lib.b200_last_error()
    assert lib.b200_pack_w8g(p, p, p, 256, 256, 64, p, None) == -1 and b"group" in lib.b200_last_error()
    # the reduce-scatter GEMM has no g64 / g32 instances: rejected on the host
    for fmt in (_lib.B200_FMT_INT4_G64, _lib.B200_FMT_INT4_G32):
        args = (fmt, 0, p, 32, 512, 4096, p, None, None, p, p, 4096, 0)
        assert lib.b200_wo_gemm_rs(*args, regs, 1 << 19, 0, 2, None) == -1 and b"group-64 / group-32" in lib.b200_last_error()


def test_w4_format_maps_groups_to_blob_formats():
    K, N = 512, 64
    s, zs = torch.rand(K // 32, N).half(), torch.rand(K // 32, N).half()
    assert ops.w4_format(K, 32, s, zs)[:2] == (_lib.B200_FMT_INT4_G32, 32)
    assert ops.w4_format(K, 64, s[:8], zs[:8])[:2] == (_lib.B200_FMT_INT4_G64, 64)
    assert ops.w4_format(K, 128, s[:4], zs[:4])[:2] == (_lib.B200_FMT_INT4, 128)
    for group, rows in ((256, 2), (512, 1), (-1, 1)):       # multiples of 128 and per-channel: group 128, rows repeated
        fmt, g, s2, z2 = ops.w4_format(K, group, s[:rows], zs[:rows])
        assert (fmt, g) == (_lib.B200_FMT_INT4, 128) and s2.shape == (4, N) and z2.shape == (4, N)
        rep = (K // rows) // 128
        assert torch.equal(s2, s[:rows].repeat_interleave(rep, 0)) and torch.equal(z2, zs[:rows].repeat_interleave(rep, 0))
    with pytest.raises(_lib.B200Error, match="group 64"):
        ops.w4_format(K, 64, s, zs)                         # 16 rows of scales do not make group 64 over K = 512


def _dense_from_unpacked(q_packed, zs, scales):
    group = q_packed.shape[0] // scales.shape[0]
    b = q_packed.numpy().astype(np.uint8)
    q = np.empty((b.shape[0], b.shape[1] * 2), np.int16)
    q[:, 0::2], q[:, 1::2] = b & 0xF, b >> 4
    q = np.where(q >= 8, q - 16, q).astype(np.float32)                       # two's-complement nibbles
    return q * np.repeat(scales.float().numpy(), group, 0) + np.repeat(zs.float().numpy(), group, 0)


def write_checkpoint(path, rng, method, group, hidden=256, heads=4, kvh=2, D=64, inter=384):
    """ckpt_util.write_checkpoint, with group -1 meaning one group per input row span (per channel, g = K of each weight)."""
    if group != -1:
        return ckpt_util.write_checkpoint(path, rng, method, hidden, heads, kvh, D, inter, group=group)
    from safetensors.torch import save_file
    shapes = dict(q=(hidden, heads * D), k=(hidden, kvh * D), v=(hidden, kvh * D), o=(heads * D, hidden), gate=(hidden, inter),
                  up=(hidden, inter), down=(inter, hidden))
    tensors, dense, names = {}, {}, {}
    for key, (K, N) in shapes.items():
        names[key] = f"model.layers.0.{key}"
        t, dense[key] = ckpt_util.make_layer(rng, method, K, N, group=K)
        tensors.update({f"{names[key]}.{sfx}": v for sfx, v in t.items()})
    save_file(tensors, path)
    return names, dense


@pytest.mark.parametrize("group", [32, 64, -1])
@pytest.mark.parametrize("method", ["gptq", "awq"])
def test_groupwise_checkpoint_at_other_groups_unpacks_to_its_dense_meaning(tmp_path, method, group):
    rng = np.random.default_rng(11)
    path = str(tmp_path / "layer.safetensors")
    names, dense = write_checkpoint(path, rng, method, group)
    ld = B200Loader(CheckpointReader(path), QuantConfig(method, group_size=group), device="cpu")
    q_packed, zs, scales = ld.groupwise_tensors([names["q"], names["k"], names["v"]])
    assert scales.shape[0] == (1 if group == -1 else 256 // group)
    np.testing.assert_allclose(_dense_from_unpacked(q_packed, zs, scales), np.concatenate([dense["q"], dense["k"], dense["v"]], 1),
                               atol=2e-3, rtol=2e-3)
    # FFN with the inter size padded from 384 to 512: w13 gains zero output columns per half, w2 zero input rows
    w13 = _dense_from_unpacked(*ld.groupwise_tensors([names["gate"], names["up"]], pad_out=512))
    assert w13.shape == (256, 1024) and np.all(w13[:, 384:512] == 0) and np.all(w13[:, 896:] == 0)
    np.testing.assert_allclose(w13[:, :384], dense["gate"], atol=2e-3, rtol=2e-3)
    np.testing.assert_allclose(w13[:, 512:896], dense["up"], atol=2e-3, rtol=2e-3)
    q_packed, zs, scales = ld.groupwise_tensors([names["down"]], pad_in=512)
    assert q_packed.shape[0] == 512 and scales.shape[0] == (1 if group == -1 else 512 // group)   # per channel: still one row
    w2 = _dense_from_unpacked(q_packed, zs, scales)
    if group == -1:
        # one zero point per column covers the padded rows too: they hold the weight of q = 0, not zero (as in the reference,
        # whose padding keeps the single row); they only ever meet the padded inter columns of w13, which are exact zeros
        assert np.all(w2[384:] == w2[384:385])
    else:
        assert np.all(w2[384:] == 0)
    np.testing.assert_allclose(w2[:384], dense["down"], atol=2e-3, rtol=2e-3)


@pytest.mark.parametrize("method", ["gptq", "awq"])
def test_per_channel_expansion_equals_a_g128_checkpoint_with_repeated_rows(method):
    """A per-channel layer stored as group 128 with every zero / scale row repeated means the same weights: the loader's
    tensors after w4_format's expansion are those of that g128 checkpoint, bit for bit."""
    rng = np.random.default_rng(3)
    K, N = 512, 256
    t, _ = ckpt_util.make_layer(rng, method, K, N, group=K)
    impl = B200Impl("cpu")
    gptq, awq = method == "gptq", method == "awq"
    q_pc, zs_pc, s_pc = impl.unpack_groupwise(t["qweight"], t["qzeros"], t["scales"], gptq, awq)
    fmt, g, s_x, zs_x = ops.w4_format(K, -1, s_pc, zs_pc)
    # the explicit g128 checkpoint: zeros are packed along N, so repeat the packed rows
    q128, zs128, s128 = impl.unpack_groupwise(t["qweight"], t["qzeros"].repeat_interleave(4, 0), t["scales"].repeat_interleave(4, 0),
                                              gptq, awq)
    assert (fmt, g) == (_lib.B200_FMT_INT4, 128)
    assert torch.equal(q_pc, q128)
    assert torch.equal(s_x.view(torch.int16), s128.view(torch.int16)) and torch.equal(zs_x.view(torch.int16), zs128.view(torch.int16))


def test_preprocess_rejects_groups_it_cannot_serve():
    impl = B200Impl("cpu")
    K, N = 256, 64
    q4 = torch.zeros(K, N // 2, dtype=torch.uint8)
    with pytest.raises(ValueError, match="group size 16"):
        impl.preprocess_weights_for_mixed_gemm(q4, torch.quint4x2, scales=torch.ones(K // 16, N).half(),
                                               zeros_x_scales=torch.zeros(K // 16, N).half())
    with pytest.raises(ValueError, match="group size K/3"):
        impl.preprocess_weights_for_mixed_gemm(q4, torch.quint4x2, scales=torch.ones(3, N).half(), zeros_x_scales=torch.zeros(3, N).half())
    q8 = torch.zeros(K, N, dtype=torch.int8)
    with pytest.raises(ValueError, match="group size 64"):
        impl.preprocess_weights_for_mixed_gemm(q8, torch.int8, scales=torch.ones(K // 64, N).half(),
                                               zeros_x_scales=torch.zeros(K // 64, N).half())
