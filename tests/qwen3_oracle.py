"""Whole-decode-step parity for Qwen3 layers (ModelConfig.qk_norm): tests/step_oracle.py's op-by-op CPU oracle with one more
stage, orc.qk_rmsnorm of the qkv rows with the layer's q_norm / k_norm gammas between the qkv GEMM and the rope append.
Layers without gammas compose exactly as step_oracle.oracle_step does."""
import dataclasses

import numpy as np
import torch

from oracle import oracle as orc
from rtp_llm_b200 import ops, rope
from rtp_llm_b200.decode_step import TINY_QWEN3, DecodeStep
from tests.spec_oracle import spec_verify_np
from tests.step_oracle import bits, gemm


def oracle_step(model: DecodeStep, kv_before):
    """The logits of one step of `model` (a DecodeStep, or any object with the attributes read here), op by op on the CPU:
    step_oracle.oracle_step's composition (q_len tokens per sequence, the rope spec under the seams' rule, act-order gathers),
    with QK-norm of q and k heads before the append in every layer that carries "q_norm" / "k_norm"."""
    cfg, B, n, Hq, Hkv, D, T = model.cfg, model.B, model.q_len, model.Hq, model.Hkv, model.D, model.cfg.tokens_per_block
    spec = model.rope_spec
    seq = model.seq_lens_h.numpy()
    pl = orc.convert_block_table(model.block_ids_h.numpy())
    if rope.is_plain_base(spec, D):
        def append(qkv, pool, s):
            return orc.rope_append(qkv, pool, pl, s, Hq, Hkv, D, T, spec.base)
    else:
        fields = {f: getattr(spec, f) for f, _ in orc.RopeConfig._fields_}
        table = rope.build_table(spec)
        cache = None if table is None else table.numpy()

        def append(qkv, pool, s):
            return orc.rope_append_ex(qkv, pool, pl, s, Hq, Hkv, D, T, fields, cos_sin_cache=cache)
    resid = bits(model.embed)[model.ids_h.numpy().reshape(-1)]
    proj = None
    for li, L in enumerate(model.layers):
        P = {k: v.numpy() for k, v in L.get("perm", {}).items()}
        gathered = lambda t, k: t[:, P[k]] if P else t  # noqa: E731
        if li == 0:
            x, _ = orc.add_rmsnorm(resid, None, bits(L["ln1"]), cfg.eps)
        else:
            x, resid = orc.add_rmsnorm(proj, resid, bits(L["ln1"]), cfg.eps)
        qkv = gemm(gathered(x, "qkv"), L["ref"]["qkv"])
        if "q_norm" in L:
            qkv = orc.qk_rmsnorm(qkv, bits(L["q_norm"]), bits(L["k_norm"]), Hq, Hkv, D, cfg.eps)
        qkv = qkv.reshape(B, n, -1)
        pool, qs = kv_before[li], []
        for j in range(n):
            qj, pool = append(np.ascontiguousarray(qkv[:, j]), pool, seq + j)
            qs.append(qj)
        a = np.stack([orc.paged_decode_attn(qs[j].reshape(B, Hq, D), pool, pl, seq + j, Hq, Hkv, D, T) for j in range(n)],
                     axis=1).reshape(B * n, -1)
        proj = gemm(gathered(a, "o"), L["ref"]["o"])
        x, resid = orc.add_rmsnorm(proj, resid, bits(L["ln2"]), cfg.eps)
        act = orc.silu_and_mul(gemm(gathered(x, "w13"), L["ref"]["w13"]))
        proj = gemm(gathered(act, "w2"), L["ref"]["w2"])
    x, resid = orc.add_rmsnorm(proj, resid, bits(model.final_ln), cfg.eps)
    return orc.from_bits(gemm(x, model.lm_head_ref), False)


def check_step(cfg=TINY_QWEN3, quant=None, batch=3, ctx=40, mode="eager", q_len=1, act_order=False, seed=1,
               dev=torch.device("cuda:0")) -> float:
    """step_oracle.check_step against this module's oracle_step: DecodeStep(cfg with `quant`, ragged lengths, reference weights
    kept), one step in `mode` ("eager", or any of "graph", "pdl", "program" together), logits within 3e-2 * rms + 3e-2, greedy
    tokens equal to the oracle's argmax wherever its top-2 margin exceeds twice that error, and for q_len > 1 the verifier's
    out_tokens / accepted on the step's own greedy rows. Returns the max |logit error|."""
    if quant is not None:
        cfg = dataclasses.replace(cfg, quant=quant)
    model = DecodeStep(cfg, batch, ctx, dev, keep_reference=True, ragged=True, seed=seed, pdl="pdl" in mode, act_order=act_order,
                       q_len=q_len)
    try:                                    # DecodeStep(pdl=True) switched PDL on library-wide
        kv_before = [bits(L["kv"]) for L in model.layers]
        if "program" in mode:
            model.build_program()
            assert model.prog.num_ops > 0, "nothing was fused into the persistent kernel"
        if "graph" in mode:                 # capture() runs the step (appends K/V) before recording it: the append is idempotent
            model.capture()
            model.replay()
        else:
            model.run()
        torch.cuda.synchronize(dev)
    finally:
        ops.set_pdl(False)
    got = model.logits.float().cpu().numpy()
    exp = oracle_step(model, kv_before)
    scale = float(np.sqrt((exp ** 2).mean()))
    err = float(np.abs(got - exp).max())
    assert np.isfinite(got).all()
    assert err <= 3e-2 * scale + 3e-2, f"logits differ: max err {err} vs rms {scale}"
    nxt = model.next_ids.cpu().numpy()
    oa = orc.argmax(exp)
    srt = np.sort(exp, axis=-1)
    sure = srt[:, -1] - srt[:, -2] > 2 * err + 1e-6
    assert (nxt[sure] == oa[sure]).all(), (nxt, oa)
    if q_len > 1:
        eo, ea = spec_verify_np(model.ids_h[:, 1:].numpy(), target_ids=nxt.reshape(model.B, q_len))
        np.testing.assert_array_equal(model.accepted.cpu().numpy(), ea)
        np.testing.assert_array_equal(model.out_tokens.cpu().numpy(), eo)
    return err
