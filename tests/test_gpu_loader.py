"""Checkpoint -> kernel layout -> GEMM on an H100 (loader.py + device.py + linear.py): the GEMM through the loaded weights must
equal X . W for the dense weight the checkpoint means; kernels survive the copies the reference loader makes."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.linear import B200WeightOnlyLinear  # noqa: E402
from rtp_llm_b200.loader import B200Loader, CheckpointReader, QuantConfig  # noqa: E402
from tests import ckpt_util  # noqa: E402

dev = torch.device("cuda")


@pytest.mark.parametrize("method", ["gptq", "awq", "int8", "none", "gptq8", "awq8"])
def test_layer_through_the_loader(tmp_path, method):
    rng = np.random.default_rng(7)
    path = str(tmp_path / "layer.safetensors")
    hidden, heads, kvh, D, inter, align = 512, 4, 2, 128, 640, 256
    bits = 8 if method.endswith("8") and method != "int8" else 4
    method = method[:-1] if bits == 8 else method
    names, dense = ckpt_util.write_checkpoint(path, rng, method, hidden, heads, kvh, D, inter, bits=bits)
    ld = B200Loader(CheckpointReader(path), QuantConfig(method, bits=bits), device=dev, align_size=align)
    L = ld.layer(names, inter=inter)
    inter_p = 768
    x = torch.from_numpy(rng.standard_normal((9, hidden)).astype(np.float32)).half().to(dev)
    ws = ops.gemm_workspace(16, [(hidden, 2 * inter_p), (inter_p, hidden), (hidden, (heads + 2 * kvh) * D)], dev)
    tol = dict(gptq=2e-2, awq=2e-2, int8=3e-2, none=1e-2)[method]

    def close(y, ref):
        ref = torch.from_numpy(ref).to(dev)
        assert (y.float() - ref).abs().max().item() <= tol * ref.abs().max().item() + tol

    xf = x.float().cpu().numpy()
    close(ops.wo_gemm(x, L["qkv"], ws), xf @ np.concatenate([dense["q"], dense["k"], dense["v"]], 1))
    assert L["w13_fused_silu"]
    g, u = xf @ dense["gate"], xf @ dense["up"]
    act = ops.wo_gemm(x, L["w13"], ws, silu_mul=True)
    assert tuple(act.shape) == (9, inter_p)
    close(act[:, :inter], g / (1 + np.exp(-g)) * u)
    assert float(act[:, inter:].abs().max()) == 0.0                            # padded inter columns are exact zeros
    a16 = act.float().cpu().numpy()
    close(ops.wo_gemm(act, L["w2"], ws), a16[:, :inter] @ dense["down"])


def test_kernels_survive_the_loaders_copies():
    """device_impl.py:296-298 returns kernel.contiguous().to(device); state dicts clone tensors: the blob is self-describing."""
    rng = np.random.default_rng(2)
    t, dense = ckpt_util.make_layer(rng, "awq", 256, 256)
    from rtp_llm_b200.device import B200Impl
    impl = B200Impl(dev)
    kernel, zs, scales = impl.preprocess_groupwise_weight_params(t["qweight"], t["qzeros"], t["scales"], "cuda", False, True, 4)
    copy = {"w": kernel.clone()}["w"].cpu().to(dev).contiguous()
    lin = B200WeightOnlyLinear(copy, weight_scales=scales, quant_config=type("AWQConfig", (), {"get_method": lambda self: "awq"})())
    x = torch.from_numpy(rng.standard_normal((4, 256)).astype(np.float32)).half().to(dev)
    ref = torch.from_numpy(x.float().cpu().numpy() @ dense).to(dev)
    assert (lin(x).float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 2e-2
    q8, s8 = impl.apply_int8(torch.from_numpy(dense).float(), "cuda")
    lin8 = B200WeightOnlyLinear(q8.clone(), weight_scales=s8, quant_config=type("W8", (), {"get_method": lambda self: "weightonly_int8"})())
    assert (lin8(x).float() - ref).abs().max().item() <= 3e-2 * ref.abs().max().item() + 3e-2
    with pytest.raises(Exception):
        B200WeightOnlyLinear(torch.zeros(1000, dtype=torch.uint8, device=dev), weight_scales=scales, quant_config=None)
