"""Whole-decode-step parity: the GPU step (rtp_llm_b200.decode_step.DecodeStep) against the CPU oracle composed op by op on
the same weights / page tables / inputs, in every mode of the step, with the whole-step logit tolerance and the two-launch
QK-norm composition the fused append replaces. Used by tests (-m gpu), tools and __graft_entry__.smoke()."""
import dataclasses
import types

import numpy as np
import torch

from oracle import oracle as orc
from rtp_llm_b200 import ops, rope
from rtp_llm_b200.decode_step import TINY, DecodeStep
from tests.spec_oracle import spec_verify_np

# Llama-3.1 rope on the tiny config. Llama3 keeps a rotary dim's angle below wavelength max_pos / factor2, divides it by scale
# above max_pos / factor1 and blends in between. max_pos 16 puts about three quarters of the dims at the tiny contexts'
# positions (20..70) in the blended or divided band, so the step's logit tolerance separates Llama3 from Base rotation; at
# Llama-3.1's own max_pos these short contexts would rotate almost as Base does.
TINY31 = dataclasses.replace(TINY, quant="int4", rope=rope.RopeSpec(style=rope.LLAMA3, dim=128, base=500000.0, scale=8.0,
                                                                    factor1=1.0, factor2=4.0, max_pos=16))


def bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def gemm(x_bits, ref, is_bf16=False):
    fmt, w, s, zs = ref
    if fmt == "int4":
        return orc.dequant_gemm(x_bits, "int4", w.numpy(), scales=bits(s), zeros_x_scales=bits(zs), group=128, is_bf16=is_bf16)
    if fmt == "int8g":
        return orc.dequant_gemm(x_bits, "int8g", w.numpy(), scales=bits(s), zeros_x_scales=bits(zs), group=128, is_bf16=is_bf16)
    if fmt == "int8":
        return orc.dequant_gemm(x_bits, "int8", w.numpy(), scales=bits(s), is_bf16=is_bf16)
    return orc.dequant_gemm(x_bits, "f16", bits(w), is_bf16=is_bf16)


def oracle_step(model: DecodeStep, kv_before):
    """The logits of one step of `model` (a DecodeStep, or any object with the attributes read here), op by op on the CPU.
    - q_len tokens per sequence: every token's K/V is appended at seq + j before any query attends; query j attends up to
      seq + j.
    - the step's rope spec, under the seams' rule: the b200_rope_append oracle for a plain Base spec, else the full rope
      contract with the spec's fields and its cos/sin table.
    - act-order (a layer with "perm"): x[:, perm] before qkv / w13, attn[:, perm] before o, and the SiLU*mul output in w2's
      row order before w2 (what the folded w13 emits). L["ref"] holds the sorted qkv / o / w2 and the checkpoint-order w13.
    - QK-norm (a layer with "q_norm" / "k_norm", ModelConfig.qk_norm): orc.qk_rmsnorm of the q and k heads of the qkv rows
      between the qkv GEMM and the append."""
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


def device_state(model: DecodeStep):
    """The fields oracle_step reads, with the inputs taken from the step's device state: for a step whose state advances
    (beam, sampling), the state the next step starts from."""
    return types.SimpleNamespace(cfg=model.cfg, B=model.B, q_len=model.q_len, Hq=model.Hq, Hkv=model.Hkv, D=model.D,
                                 rope_spec=model.rope_spec, seq_lens_h=model.seq_lens.cpu(), block_ids_h=model.block_ids.cpu(),
                                 ids_h=model.ids.cpu(), embed=model.embed, layers=model.layers, final_ln=model.final_ln,
                                 lm_head_ref=model.lm_head_ref)


def logit_error(got, exp, mask=None):
    """(max |got - exp|, the whole-step tolerance 3e-2 * rms(exp) + 3e-2) over the elements `mask` selects (all without one).
    The one statement of the tolerance: check_logits asserts it, tools/tp_check.py reports it."""
    if mask is not None:
        got, exp = got[mask], exp[mask]
    return float(np.abs(got - exp).max()), 3e-2 * float(np.sqrt((exp ** 2).mean())) + 3e-2


def check_logits(got, exp, mask=None) -> float:
    """Asserts the logits `got` finite and within logit_error's tolerance of the oracle's `exp` over the elements `mask`
    selects; returns the max |error|."""
    err, bound = logit_error(got, exp, mask)
    finite = np.isfinite(got if mask is None else got[mask]).all()
    assert finite and err <= bound, f"logits differ: max err {err} vs bound {bound}"
    return err


class TwoLaunchStep(DecodeStep):
    """The composition the fused QK-norm append replaces: qk_rmsnorm in place on qkv, then rope.rope_append without QK-norm."""

    def _rope_append(self, L):
        ops.qk_rmsnorm(self.qkv, L["q_norm"], L["k_norm"], self.Hq, self.Hkv, self.D, self.cfg.eps)
        rope.rope_append(self.rope_spec, self.qkv, L["kv"], self.page_list, self.seq_lens, self.Hq, q_out=self.q, q_len=self.q_len)


def check_step(cfg=TINY, quant=None, batch=3, ctx=40, mode="eager", q_len=1, act_order=False, fuse_rope=False, seed=1,
               dev=torch.device("cuda:0")) -> float:
    """Builds DecodeStep(cfg with `quant`, ragged lengths, reference weights kept), runs one step and checks it against
    oracle_step. mode: "eager" (op by op), or any of "graph" (captured and replayed), "pdl" and "program" (recorded into a
    decode program) together. Asserts check_logits against the oracle, greedy tokens equal to the oracle's argmax wherever
    its top-2 margin exceeds twice the logit error, and for q_len > 1 the verifier's out_tokens / accepted on the step's own
    greedy rows. Returns the max |logit error|."""
    if quant is not None:
        cfg = dataclasses.replace(cfg, quant=quant)
    model = DecodeStep(cfg, batch, ctx, dev, keep_reference=True, ragged=True, seed=seed, pdl="pdl" in mode, fuse_rope=fuse_rope,
                       act_order=act_order, q_len=q_len)
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
    exp = oracle_step(model, kv_before)
    err = check_logits(model.logits.float().cpu().numpy(), exp)
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
