"""GPTQ act-order (desc_act) checkpoints on the host (no GPU): the g_idx -> row order helper, the loader's sort of the rows of
synthetic AutoGPTQ act-order checkpoints, merged parts, w2 padding, the w2 -> w13 column fold, the perm-carrying blob trailer and
the argument checks of b200_permute_cols. The kernel side is tests/test_gpu_act_order.py."""
import ctypes

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, ops
from rtp_llm_b200.device import act_order_perm
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig
from tests import act_order_ckpt


def _signed(q_unpacked, bits):
    """The loader's q (4-bit: uint8 [K, N/2] two's-complement nibbles; 8-bit: int8 [K, N]) -> int [K, N]."""
    if bits == 8:
        return q_unpacked.numpy().astype(np.int32)
    b = q_unpacked.numpy().astype(np.int32)
    q = np.empty((b.shape[0], b.shape[1] * 2), np.int32)
    q[:, 0::2], q[:, 1::2] = b & 0xF, b >> 4
    return np.where(q >= 8, q - 16, q)


@pytest.mark.parametrize("bits,group", [(4, 128), (4, 64), (4, 32), (8, 128)])
def test_loader_sorts_rows_by_g_idx(tmp_path, bits, group):
    rng = np.random.default_rng(5)
    K, N = 512, 64
    g_idx = act_order_ckpt.act_order_g_idx(rng, K, group)
    t, dense, q_u, z, s = act_order_ckpt.make_act_order_layer(rng, K, N, g_idx, group, bits)
    from safetensors.torch import save_file
    path = str(tmp_path / "w.safetensors")
    save_file({f"w.{k}": v for k, v in t.items()}, path)
    ld = B200Loader(CheckpointReader(path), QuantConfig("gptq", bits=bits, group_size=group), device="cpu")
    q, zs, scales, perm = ld.sorted_tensors(["w"])
    perm = perm.numpy()
    assert sorted(perm.tolist()) == list(range(K))
    assert np.array_equal(g_idx[perm], np.arange(K) // group)                        # groups are contiguous after the sort
    assert np.array_equal(_signed(q, bits), q_u[perm] - (1 << (bits - 1)))            # row j = checkpoint row perm[j], exactly
    # the scale / zero*scale rows are untouched: sorted row j meets group g_idx[perm[j]] = j // group
    assert torch.equal(scales.view(torch.int16), torch.from_numpy(s).view(torch.int16))
    zs_exp = (((1 << (bits - 1)) - z) * s.astype(np.float32)).astype(np.float16)       # GPTQ stores z - 1
    assert np.array_equal(zs.numpy().view(np.uint16), zs_exp.view(np.uint16))
    # and together they mean the checkpoint's dense rows in the sorted order
    deq = _signed(q, bits) * np.repeat(scales.float().numpy(), group, 0) + np.repeat(zs.float().numpy(), group, 0)
    np.testing.assert_allclose(deq, dense[perm], atol=2e-3, rtol=2e-3)


def test_act_order_perm_trivial_and_malformed():
    K = 512
    for group in (128, 64, 32):
        assert act_order_perm(None, group, K) is None
        assert act_order_perm(torch.arange(K, dtype=torch.int32) // group, group, K) is None      # static groups / no act-order
    assert act_order_perm(torch.zeros(K, dtype=torch.int32), -1, K) is None                      # per channel
    assert act_order_perm(torch.zeros(K, dtype=torch.int32), K, K) is None
    g = torch.from_numpy(act_order_ckpt.act_order_g_idx(np.random.default_rng(1), K, 128))
    perm = act_order_perm(g, 128, K)
    assert torch.equal(g[perm], torch.arange(K) // 128)
    assert torch.equal(perm, torch.sort(g.long(), stable=True).indices)
    with pytest.raises(ValueError, match="entries"):
        act_order_perm(g[:-1], 128, K)
    bad = g.clone()
    bad[0] = 4
    with pytest.raises(ValueError, match=r"\[0, 4\)"):
        act_order_perm(bad, 128, K)
    bad[0] = -1
    with pytest.raises(ValueError, match=r"\[0, 4\)"):
        act_order_perm(bad, 128, K)
    unbalanced = g.clone()
    unbalanced[int(torch.nonzero(g == 1)[0])] = 0                                            # group 0: 129 rows, group 1: 127
    with pytest.raises(ValueError, match="exactly 128"):
        act_order_perm(unbalanced, 128, K)


def test_merged_parts_must_share_g_idx(tmp_path):
    from safetensors.torch import save_file
    rng = np.random.default_rng(2)
    K = 256
    g1, g2 = act_order_ckpt.act_order_g_idx(rng, K, 128), act_order_ckpt.act_order_g_idx(rng, K, 128)
    tensors = {}
    for name, g in (("q", g1), ("k", g1), ("v", g2), ("gate", g1), ("up", g1)):
        t, *_ = act_order_ckpt.make_act_order_layer(rng, K, 128, g)
        tensors.update({f"l.{name}.{k}": v for k, v in t.items()})
    t, *_ = act_order_ckpt.make_act_order_layer(rng, K, 128, np.arange(K) // 128)
    tensors.update({f"l.plain.{k}": v for k, v in t.items() if k != "g_idx"})
    path = str(tmp_path / "l.safetensors")
    save_file(tensors, path)
    ld = B200Loader(CheckpointReader(path), QuantConfig("gptq"), device="cpu")
    with pytest.raises(ValueError, match="l.q and l.v .*different g_idx"):
        ld.act_order(["l.q", "l.k", "l.v"])
    with pytest.raises(ValueError, match="different g_idx"):
        ld.act_order(["l.gate", "l.plain"])                  # act-order next to a part without g_idx
    assert torch.equal(ld.act_order(["l.gate", "l.up"]), act_order_perm(torch.from_numpy(g1), 128, K))
    # AWQ has no g_idx: never read
    assert B200Loader(CheckpointReader(path), QuantConfig("awq"), device="cpu").act_order(["l.q", "l.v"]) is None


def test_w2_padding_and_the_w13_fold(tmp_path):
    rng = np.random.default_rng(8)
    hidden, inter, align = 256, 384, 256
    path = str(tmp_path / "layer.safetensors")
    names, dense, gi = act_order_ckpt.write_act_order_checkpoint(path, rng, hidden, 2, 1, 128, inter)
    ld = B200Loader(CheckpointReader(path), QuantConfig("gptq"), device="cpu", align_size=align)
    q, zs, scales, perm = ld.sorted_tensors([names["down"]], pad_in=512)
    p2 = ld.act_order([names["down"]])
    assert q.shape[0] == 512 and torch.equal(perm[:inter], p2) and torch.equal(perm[inter:], torch.arange(inter, 512))
    # the padded rows stay in place as groups of their own, with zero scales and zero*scales: zero weights
    assert scales.shape[0] == 4 and float(scales[3:].abs().max()) == 0 and float(zs[3:].abs().max()) == 0
    # fold: w13's gate and up output columns in w2's row order; the padded columns keep their place
    q13, zs13, s13, perm13 = ld.sorted_tensors([names["gate"], names["up"]], pad_out=512, col_perm=p2)
    q0, zs0, s0, _ = ld.sorted_tensors([names["gate"], names["up"]], pad_out=512)
    cp = torch.cat([p2, torch.arange(inter, 512)])
    order = torch.cat([cp, cp + 512]).numpy()
    assert torch.equal(perm13, act_order_perm(torch.from_numpy(gi["w13"]), 128, hidden))
    assert np.array_equal(_signed(q13, 4), _signed(q0, 4)[:, order])
    assert torch.equal(s13, s0[:, order]) and torch.equal(zs13, zs0[:, order])


def test_column_permutation_of_packed_int4_equals_unpack_permute_repack():
    rng = np.random.default_rng(4)
    K, N = 64, 256
    packed = torch.from_numpy(rng.integers(0, 256, (K, N // 2)).astype(np.uint8))
    order = torch.randperm(N, generator=torch.Generator().manual_seed(3))
    got = ops.permute_columns(packed, order, packed_int4=True).numpy()
    full = np.empty((K, N), np.uint8)
    full[:, 0::2], full[:, 1::2] = packed.numpy() & 0xF, packed.numpy() >> 4
    full = full[:, order.numpy()]
    assert np.array_equal(got, full[:, 0::2] | (full[:, 1::2] << 4))


def test_perm_blob_trailer_round_trip_and_check():
    """[blob | perm int32 [K] | trailer] under its own magic; from_tensor recovers the perm from any copy. Old blobs keep their
    exact size."""
    K, N = 256, 128
    n = int(_lib.load().b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4, K, N))
    perm = torch.randperm(K, generator=torch.Generator().manual_seed(0))
    blob = ops._blob(n, K, perm, "cpu")
    w = ops._packed(_lib.B200_FMT_INT4, K, N, blob, 128, n, True)
    assert blob.numel() == n + 4 * K + 256 and torch.equal(w.perm.long(), perm)
    again = ops.PackedWeight.from_tensor(blob.clone())
    assert (again.fmt, again.K, again.N) == (_lib.B200_FMT_INT4, K, N) and torch.equal(again.perm.long(), perm)
    plain = ops._packed(_lib.B200_FMT_INT4, K, N, ops._blob(n, K, None, "cpu"), 128, n, False)
    assert plain.data.numel() == n + 256 and ops.PackedWeight.from_tensor(plain.data).perm is None
    old_magic = blob.clone()
    ops.PackedWeight._write_trailer(old_magic, _lib.B200_FMT_INT4, K, N, 128)
    with pytest.raises(_lib.B200Error, match="bytes"):
        ops.PackedWeight.from_tensor(old_magic)              # the perm bytes count only under the new magic
    for bad in (perm[:-1], torch.cat([perm[:-1], perm[:1]]), perm + 1):
        with pytest.raises(_lib.B200Error, match="permutation"):
            ops._blob(n, K, bad, "cpu")


def test_permute_cols_argument_checks():
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 8192)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    a, b = (p + 15) // 16 * 16, (p + 15) // 16 * 16 + 4096
    assert lib.b200_permute_cols(None, a, b, 0, 4, 64, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_permute_cols(a, None, b, 0, 4, 64, None) == -1 and b"null" in lib.b200_last_error()
    assert lib.b200_permute_cols(a, a, a, 0, 4, 64, None) == -1 and b"same buffer" in lib.b200_last_error()
    assert lib.b200_permute_cols(a, a, b, 0, 4, 60, None) == -1 and b"multiple of 8" in lib.b200_last_error()
    assert lib.b200_permute_cols(a, a, b, 0, 4, 65544, None) == -1 and b"multiple of 8" in lib.b200_last_error()
    assert lib.b200_permute_cols(a + 2, a, b, 0, 4, 64, None) == -1 and b"aligned" in lib.b200_last_error()
    assert lib.b200_permute_cols(a, a, b, 0, 0, 64, None) == 0                            # nothing to do


def test_decode_step_act_order_rejects_tp_and_unquantised_weights():
    """A row-parallel o shard would hold rows of groups that span every rank; f16 / per-column int8 weights have no groups."""
    import dataclasses
    from rtp_llm_b200.decode_step import TINY, DecodeStep
    with pytest.raises(ValueError, match="tp_size 1"):
        DecodeStep(TINY, 1, 16, torch.device("cpu"), tp_rank=0, tp_size=2, act_order=True)
    for quant in ("f16", "int8"):
        with pytest.raises(ValueError, match="int4 / int8g"):
            DecodeStep(dataclasses.replace(TINY, quant=quant), 1, 16, torch.device("cpu"), act_order=True)
