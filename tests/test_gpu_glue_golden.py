"""Our glue kernels against outputs of the CUDA kernels the reference binds (flashinfer rmsnorm / fused_add_rmsnorm /
silu_and_mul, captured with flashinfer 0.6.11.post2 on a B200 by tools/make_gpu_golden.py and re-captured bit-identically on an H100 into tests/golden/flashinfer_glue_ops.npz)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402

dev = torch.device("cuda")


def _t(a, dtype):
    return torch.from_numpy(a.copy()).view(dtype).to(dev)


@pytest.mark.parametrize("tag", ["f16_512", "f16_4096", "bf16_512", "bf16_4096"])
def test_rmsnorm_kernels_vs_flashinfer_outputs(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "flashinfer_glue_ops.npz"))
    dtype = torch.bfloat16 if tag.startswith("bf16") else torch.float16
    x, r, w = (_t(g[f"{tag}_{k}"], dtype) for k in ("x", "res", "w"))
    tol = 1.6e-2 if dtype == torch.bfloat16 else 2e-3
    y = ops.add_rmsnorm(x, None, w, 1e-6)
    torch.testing.assert_close(y.float(), _t(g[f"{tag}_rmsnorm"], dtype).float(), rtol=tol, atol=tol)
    r2 = r.clone()
    y2 = ops.add_rmsnorm(x, r2, w, 1e-6)
    assert torch.equal(r2, _t(g[f"{tag}_fused_res"], dtype))                       # stored residual: bit-exact
    exp = _t(g[f"{tag}_fused_y"], dtype)
    torch.testing.assert_close(y2.float(), exp.float(), rtol=tol, atol=tol)
    assert (y2 == exp).float().mean().item() > 0.97


@pytest.mark.parametrize("tag", ["f16", "bf16"])
def test_silu_and_mul_vs_flashinfer_outputs(golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "flashinfer_glue_ops.npz"))
    dtype = torch.bfloat16 if tag == "bf16" else torch.float16
    y = ops.silu_and_mul(_t(g[f"{tag}_gate_up"], dtype))
    exp = _t(g[f"{tag}_silu_and_mul"], dtype)
    tol = 1.6e-2 if dtype == torch.bfloat16 else 2e-3
    torch.testing.assert_close(y.float(), exp.float(), rtol=tol, atol=tol)
    assert (y == exp).float().mean().item() > 0.95
