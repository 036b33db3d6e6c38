"""b200_sample (csrc/sampling.cuh) against the sampling oracle, which is pinned to the reference's CudaSamplerTest vectors
(tests/test_sampler_oracle.py), through the C ABI on an H100."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from rtp_llm_b200 import ops  # noqa: E402

dev = torch.device("cuda")


def _t(a, dt):
    return None if a is None else torch.tensor(np.asarray(a), dtype=dt, device=dev)


def _run(lg, top_k, top_p, u, temperature=None, history=None, hist_len=None, repetition=None, presence=None, frequency=None,
         process=None):
    x = torch.tensor(lg, dtype=torch.float32, device=dev)
    ws = torch.zeros_like(x, dtype=torch.int32)
    tok, tprob, probs = ops.sample(x, _t(top_k, torch.int32), _t(top_p, torch.float32), _t(u, torch.float32),
                                   temperature=_t(temperature, torch.float32), history=_t(history, torch.int32),
                                   hist_len=_t(hist_len, torch.int32), repetition=_t(repetition, torch.float32),
                                   presence=_t(presence, torch.float32), frequency=_t(frequency, torch.float32),
                                   process=_t(process, torch.uint8), count_ws=ws, want_probs=True)
    torch.cuda.synchronize()
    assert int(ws.abs().sum()) == 0, "count workspace not left clean"
    return tok.cpu().numpy(), tprob.cpu().numpy(), x.cpu().numpy(), probs.cpu().numpy()


def test_reference_vectors_through_the_kernel():
    lg = np.array([0, 0, 0, 0.1, 0.2, 0.3, 0, 0, 0, 0.01, 0.987, 0.887, 0.99999, 0.1, 0.2, 0.3, 0, 0, 0.99, 0.989, 0.221, 0, 0, 0.1,
                   0.2, 0.321, 0, 0.4432, 0.44, 0.01, 0.221, 0, 0, 0.1, 0.2, 0.321, 0, 0.4432, 0.44, 0.01], np.float32).reshape(4, 10)
    tok, _, _, _ = _run(lg, [1, 1, 1, 1], [1.0] * 4, [0.3, 0.9, 0.1, 0.7], temperature=[1.0, 10.0, 1.0, 10.0])
    assert tok.tolist() == [5, 2, 7, 7]                                        # CudaSamplerTest.cc:564-567
    lg2 = np.tile(np.array([0.01, 0.8, 0.98, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7], np.float32), (4, 1))
    tok, _, _, probs = _run(lg2, [2] * 4, [1.0] * 4, [0.9, 0.1, 0.2, 0.3], temperature=[2.0, 2.0, 4.0, 4.0], process=[0, 1, 0, 1])
    assert tok.tolist() == [2, 1, 1, 1]
    np.testing.assert_allclose(probs[:, 1], [0.455121, 0.477515, 0.455121, 0.488752], atol=1e-3)   # :1046-1050


@pytest.mark.parametrize("vocab", [1000, 32000, 128256])
def test_kernel_matches_oracle_on_random_rows(vocab):
    rng = np.random.default_rng(vocab)
    B, L = 9, 300
    lg = (rng.standard_normal((B, vocab)) * 3).astype(np.float32)
    hist = rng.integers(0, vocab, (B, L)).astype(np.int32)
    hist[:, ::7] = hist[:, :1]                                                   # repeated tokens: counts > 1
    hl = rng.integers(1, L + 1, B).astype(np.int32)
    top_k = np.array([1, 0, 5, 50, 0, 1000, 2, 0, 40], np.int32)
    top_p = np.array([1.0, 1.0, 1.0, 0.9, 0.8, 0.5, 0.3, 0.0, 0.95], np.float32)
    u = rng.random(B).astype(np.float32) * 0.98 + 0.01
    kw = dict(temperature=(rng.random(B) + 0.5).astype(np.float32), history=hist, hist_len=hl,
              repetition=np.array([1.0, 1.3, 1.0, 2.0, 1.1, 1.0, 1.5, 1.0, 1.2], np.float32),
              presence=np.array([0, 0.5, 0, 0.1, 0, 0.2, 0, 0, 0.3], np.float32),
              frequency=np.array([0, 0, 0.3, 0.1, 0, 0, 0.2, 0, 0.1], np.float32), process=np.array([1, 1, 1, 1, 0, 1, 1, 1, 1], np.uint8))
    tok, tprob, soft, probs = _run(lg, top_k, top_p, u, **kw)
    etok, etprob, esoft, eprobs = orc.sample(lg, top_k, top_p, u, **kw)
    np.testing.assert_allclose(soft, esoft, rtol=2e-4, atol=1e-9)              # softmax after temperature + penalties
    # the kept set must be identical wherever no probability sits within rounding of the threshold
    kept, ekept = probs > 0, eprobs > 0
    for r in range(B):
        if not np.array_equal(kept[r], ekept[r]):
            thr = eprobs[r][ekept[r]].min()
            near = np.abs(esoft[r] / esoft[r][ekept[r]].sum() - thr) < 1e-5 * thr + 1e-12
            assert np.array_equal(kept[r] & ~near, ekept[r] & ~near), f"row {r}: kept sets differ away from the threshold"
    np.testing.assert_allclose(probs, eprobs, rtol=1e-3, atol=1e-7)
    # the draw: equal tokens unless the uniform lands within float rounding of a CDF step
    for r in range(B):
        if tok[r] != etok[r]:
            cdf = np.cumsum(eprobs[r].astype(np.float64))
            assert np.min(np.abs(cdf - u[r])) < 1e-5, f"row {r}: token {tok[r]} vs oracle {etok[r]} with u well inside a CDF step"
    assert (tok == etok).mean() >= 0.8
    np.testing.assert_allclose(tprob, probs[np.arange(B), tok], rtol=1e-5)


def test_draws_follow_the_renormalised_distribution():
    """Distribution-level check in the spirit of the reference's own accuracy test (CudaSamplerTest.cc:143-147: l1 < 0.08)."""
    rng = np.random.default_rng(0)
    V, N = 64, 4096
    row = (rng.standard_normal(V) * 2).astype(np.float32)
    lg = np.tile(row, (N, 1))
    tok, _, _, probs = _run(lg, [12] * N, [0.9] * N, rng.random(N).astype(np.float32))
    emp = np.bincount(tok, minlength=V) / N
    assert np.abs(emp - probs[0]).sum() < 0.08 and set(np.flatnonzero(emp)) <= set(np.flatnonzero(probs[0]))
