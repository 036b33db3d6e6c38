#!/usr/bin/env python
"""Step-level A/B of the decode step's modes (developer tool, runs on the GPU). A preset builds two or more arms per batch,
each a step captured in a CUDA graph with PDL at --ctx tokens; the first arm is the baseline.

  act-order  Llama-3-8B INT4: plain, then act_order=True (three gathers per layer; w2's order is folded into w13)
  spec       Llama-3-8B INT4 (--model llama31: Llama-3.1-8B with its Llama3 rope): q_len 1, 2, 4 with batch * q_len <= 128
  beam       Llama-3-8B INT4: the greedy step at batch * W rows, the beam step with b200_paged_decode_attn on every beam's row
             (PerRowBeamStep), the beam step as it is (W beams per request, --ngram ban; the beam attention kernel when the
             rows fit), with --eos the beam step that also keeps the finished hypotheses (eos_id set), and the fork alone as a
             graph of DecodeStep.fork()
  sample     Llama-3-8B INT4: greedy, then sampled (temperature 0.8, top-k 50, top-p 0.9, repetition 1.1, the drawn token's
             log-prob and the top 5)
  qwen3      Qwen3-8B INT4: qk_rmsnorm, then the plain rope launch (TwoLaunchStep), against the fused QK-norm append
  tree       Llama-3-8B INT4: per q_len 4 and 8 with batch * q_len <= 128, the chain verification step, then the token-tree
             step on a binary tree of q_len nodes (tree attention, spec_verify_tree and the K/V compaction); with
             --draft-probs instead the sampled tree step (temperature 0.8, top-k 50, top-p 0.9) without and with draft rows
             (draft_probs=True: b200_spec_verify_tree_draft; rows of dense random softmaxes, so the root's children are
             rejected and each rejection is a pass over the vocabulary)
  prefix     Llama-3-8B INT4: the shared-prefix step (1024 prompt tokens shared by groups of 8 requests) with
             b200_paged_decode_attn on every row, then with b200_paged_decode_attn_prefix for groups of 8 and of 32
             (PrefixStep forces the kernel either way); prints which kernel attention.prefix_rows_fit picks
  constrain  Llama-3-8B INT4: greedy, greedy with a 50 % random token bitmask and 300 logit_bias entries per row, sampled
             (temperature 0.8, top-k 50, top-p 0.9), sampled with the same constraints

Every run visits the arms in turn. Per arm: restart the steps whose state advances (beam, sampled) from the prompt with
upload_inputs(), replay --warmup times, restart again, then time --iters replays with CUDA events and synchronise. An
advancing step's prompt holds ctx - max_new_tokens tokens, with max_new_tokens = max(iters, warmup) + 8: room for the longest
run between two restarts, plus the 8 spare steps the beam and sampled numbers in README.md and DESIGN.md were measured with.

Prints the card, its power limit and SM clock from the same run, then per batch and arm the median, min and max ms/step
over --runs, native launches per step, and the difference to the baseline, t - t0 in µs and t / t0 - 1. For spec, t / t0 - 1
is the break-even number of accepted drafts per verification step. --out writes the same numbers as JSON."""
import argparse
import dataclasses
import json
import os
import statistics
import subprocess
import sys
from typing import Callable, Optional, Tuple

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.attention import prefix_rows_fit  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, LLAMA31_8B, QWEN3_8B, DecodeStep, SamplingParams  # noqa: E402
from tests.step_oracle import TwoLaunchStep  # noqa: E402
from tests.test_gpu_beam_attn import PerRowBeamStep  # noqa: E402


@dataclasses.dataclass
class Arm:
    name: str
    replay: Callable[[], None]
    launches: Optional[int]                 # native launches per step; None for an arm of torch ops only
    resets: Tuple[DecodeStep, ...] = ()     # steps whose state advances with every replay


def step_arm(name: str, model: DecodeStep) -> Arm:
    launches = model.launches_per_step()    # one eager step; capture() then restarts an advancing step from its prompt
    model.capture()
    return Arm(name, model.replay, launches, (model,) if model.advances else ())


def max_new_tokens(a) -> int:
    return max(a.iters, a.warmup) + 8


def act_order_arms(a, cfg, B, dev):
    return [step_arm(name, DecodeStep(cfg, B, a.ctx, dev, pdl=True, act_order=ao)) for name, ao in (("plain", False),
                                                                                                    ("act_order", True))]


def spec_arms(a, cfg, B, dev):
    return [step_arm(f"q_len {n}", DecodeStep(cfg, B, a.ctx, dev, pdl=True, q_len=n)) for n in (1, 2, 4) if B * n <= 128]


def beam_arms(a, cfg, B, dev):
    W = a.beam_width
    greedy = step_arm(f"greedy B{B * W}", DecodeStep(cfg, B * W, a.ctx, dev, pdl=True))
    kw = dict(pdl=True, beam_width=W, no_repeat_ngram=a.ngram, max_new_tokens=max_new_tokens(a))
    per_row = step_arm(f"beam W{W} per row", PerRowBeamStep(cfg, B, a.ctx, dev, **kw))
    model = DecodeStep(cfg, B, a.ctx, dev, **kw)
    beam = step_arm(f"beam W{W}", model)
    model.replay()                          # beam_out holds a real selection for the fork graph to replay
    hyps = []
    if a.eos:                               # EOS = request 0's best candidate at step 1: hypotheses enter from the first step
        eos = int(model.beam_out["cand_token"][0, 0])
        print(f"B{B} beam W{W} + hyps: eos_id {eos}", flush=True)
        hyps = [step_arm(f"beam W{W} + hyps", DecodeStep(cfg, B, a.ctx, dev, pdl=True, beam_width=W, no_repeat_ngram=a.ngram,
                                                         max_new_tokens=max_new_tokens(a), eos_id=eos))]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model.fork()
    torch.cuda.current_stream().wait_stream(s)
    fork = torch.cuda.CUDAGraph()
    with torch.cuda.graph(fork):
        model.fork()
    model.upload_inputs()
    torch.cuda.synchronize()
    return [greedy, per_row, beam] + hyps + [Arm("fork", fork.replay, None, (model,))]


def sample_arms(a, cfg, B, dev):
    sp = SamplingParams(temperature=0.8, top_k=50, top_p=0.9, repetition=1.1, seed=1)
    return [step_arm("greedy", DecodeStep(cfg, B, a.ctx, dev, pdl=True)),
            step_arm("sampled", DecodeStep(cfg, B, a.ctx, dev, pdl=True, sampling=sp, logprobs=5,
                                           max_new_tokens=max_new_tokens(a)))]


class ConstrainedStep(DecodeStep):
    """A step that sets its A/B constraints (ab_constraints: set_constraints' arguments) again after every upload_inputs(),
    which would otherwise reset it to unconstrained."""
    ab_constraints = None

    def upload_inputs(self):
        super().upload_inputs()
        if self.ab_constraints is not None:
            self.set_constraints(*self.ab_constraints)


def constrain_arms(a, cfg, B, dev):
    sp = SamplingParams(temperature=0.8, top_k=50, top_p=0.9, seed=1)
    arms = []
    for name, kw in (("greedy", {}), ("sampled", dict(sampling=sp, max_new_tokens=max_new_tokens(a)))):
        arms.append(step_arm(name, DecodeStep(cfg, B, a.ctx, dev, pdl=True, **kw)))
        model = ConstrainedStep(cfg, B, a.ctx, dev, pdl=True, token_bitmask=True, logit_bias_capacity=300 * B, **kw)
        g = torch.Generator().manual_seed(B)
        mask = torch.randint(-2 ** 31, 2 ** 31, model.bitmask_h.shape, generator=g, dtype=torch.int64).to(torch.int32)
        bias = [dict(zip(torch.randperm(model.vocab, generator=g)[:300].tolist(), torch.randn(300, generator=g).tolist()))
                for _ in range(B)]
        model.ab_constraints = (mask, bias)
        model.upload_inputs()
        arms.append(step_arm(f"{name} + constraints", model))
    return arms


class PrefixStep(DecodeStep):
    """The shared-prefix step with its attention forced: b200_paged_decode_attn_prefix (prefix True) or b200_paged_decode_attn
    on every row (False), whatever attention.prefix_rows_fit says."""

    def __init__(self, *args, prefix: bool, **kw):
        self.force_prefix = prefix
        super().__init__(*args, **kw)

    def upload_inputs(self):
        super().upload_inputs()
        self.use_prefix = self.force_prefix


def prefix_arms(a, cfg, B, dev):
    kw = dict(pdl=True)
    models = [PrefixStep(cfg, B, a.ctx, dev, shared_prefix=(8, 1024), prefix=False, **kw)]
    models += [PrefixStep(cfg, B, a.ctx, dev, shared_prefix=(n, 1024), prefix=True, **kw) for n in (8, 32)]
    arms = [step_arm(name, m) for name, m in zip(("per row, groups of 8", "prefix kernel, groups of 8",
                                                   "prefix kernel, groups of 32"), models)]
    for m in models:
        offs, _, shared, mm = m.chunks
        fit = prefix_rows_fit(m.Hkv, shared.numel(), float(shared.float().mean()), mm)
        print(f"B{B} {m.shared_prefix}: {shared.numel()} chunks of up to {mm} rows; attention.prefix_rows_fit picks "
              f"{'the prefix kernel' if fit else 'the per-row kernel'}", flush=True)
    return arms


def tree_arms(a, cfg, B, dev):
    arms = []
    for n in (4, 8):
        if B * n <= 128:
            binary = [-1] + [(j - 1) // 2 for j in range(1, n)]
            if a.draft_probs:
                sp = SamplingParams(temperature=0.8, top_k=50, top_p=0.9, seed=1)
                kw = dict(pdl=True, q_len=n, tree=binary, sampling=sp)
                arms.append(step_arm(f"tree q_len {n} sampled", DecodeStep(cfg, B, a.ctx, dev, **kw)))
                model = DecodeStep(cfg, B, a.ctx, dev, draft_probs=True, **kw)
                g = torch.Generator(device=dev).manual_seed(n)
                model.set_draft_probs(torch.softmax(torch.randn(B, n, model.vocab, generator=g, device=dev), -1))
                arms.append(step_arm(f"tree q_len {n} sampled + draft rows", model))
                continue
            arms.append(step_arm(f"chain q_len {n}", DecodeStep(cfg, B, a.ctx, dev, pdl=True, q_len=n)))
            arms.append(step_arm(f"tree q_len {n}", DecodeStep(cfg, B, a.ctx, dev, pdl=True, q_len=n, tree=binary)))
    return arms


def qwen3_arms(a, cfg, B, dev):
    return [step_arm("norm + rope", TwoLaunchStep(cfg, B, a.ctx, dev, pdl=True)),
            step_arm("fused", DecodeStep(cfg, B, a.ctx, dev, pdl=True))]


# name: arms, default batches, timed replays per run, warm-up replays
PRESETS = {"act-order": (act_order_arms, [32], 100, 10), "spec": (spec_arms, [8, 16, 32], 50, 3),
           "beam": (beam_arms, [8], 20, 3), "sample": (sample_arms, [8, 32], 20, 3), "qwen3": (qwen3_arms, [8, 16, 32], 100, 10),
           "constrain": (constrain_arms, [8, 32], 50, 5), "tree": (tree_arms, [8, 16, 32], 50, 3), "prefix": (prefix_arms, [32, 64], 50, 5)}
MODELS = {"llama3": LLAMA3_8B, "llama31": LLAMA31_8B}


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="preset", required=True)
    for name, (arms, batch, iters, warmup) in PRESETS.items():
        p = sub.add_parser(name, help=f"the {name} arms (see above)")
        p.add_argument("--batch", type=int, nargs="+", default=batch, help="batch sizes, one A/B each (default %(default)s)")
        p.add_argument("--ctx", type=int, default=2048, help="context length (default %(default)s)")
        p.add_argument("--runs", type=int, default=5, help="runs, each visiting every arm (default %(default)s)")
        p.add_argument("--iters", type=int, default=iters, help="timed replays per run and arm (default %(default)s)")
        p.add_argument("--warmup", type=int, default=warmup, help="warm-up replays before them (default %(default)s)")
        p.add_argument("--out", help="write the results as JSON to this file")
        if name == "spec":
            p.add_argument("--model", choices=sorted(MODELS), default="llama3")
        if name == "tree":
            p.add_argument("--draft-probs", action="store_true", help="the sampled tree step without and with draft rows")
        if name == "beam":
            p.add_argument("--beam-width", type=int, default=4)
            p.add_argument("--ngram", type=int, default=0, help="no-repeat-ngram size of the beam step (default 0: off)")
            p.add_argument("--eos", action="store_true", help="add the beam step with finished-hypothesis tracking (eos_id: "
                                                              "request 0's best candidate at step 1)")
        p.set_defaults(arms=arms)
    a = ap.parse_args(argv)
    a.cfg = QWEN3_8B if a.preset == "qwen3" else MODELS[getattr(a, "model", "llama3")]
    return a


def smi(fields: str) -> str:
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip() or "unknown"


def time_arm(arm: Arm, iters: int, warmup: int) -> float:
    for m in arm.resets:
        m.upload_inputs()
    for _ in range(warmup):
        arm.replay()
    for m in arm.resets:
        m.upload_inputs()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(iters):
        arm.replay()
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / iters


def main(argv=None):
    a = parse(argv)
    if not torch.cuda.is_available():
        sys.exit(f"step_ab {a.preset}: needs a CUDA device")
    ops.device_check(0)
    dev = torch.device("cuda:0")
    card = smi("name,power.limit,clocks.sm,clocks.max.sm")
    print(f"{torch.cuda.get_device_name(0)}; name, power limit, SM clock, max SM clock: {card}")
    print(f"{a.preset}: {a.cfg.name} {a.cfg.quant} ctx {a.ctx}, CUDA graph + PDL, {a.runs} runs x {a.iters} replays after "
          f"{a.warmup} warm-ups, arms alternating", flush=True)
    res = dict(device=torch.cuda.get_device_name(0), nvidia_smi_name_power_limit_sm_clock=card, preset=a.preset,
               model=a.cfg.name, ctx=a.ctx, runs=a.runs, iters=a.iters, warmup=a.warmup, batches=[])
    if a.preset == "beam":
        res.update(beam_width=a.beam_width, ngram=a.ngram, eos=a.eos)
    if a.preset == "tree":
        res.update(draft_probs=a.draft_probs)
    try:
        for B in a.batch:
            arms = a.arms(a, a.cfg, B, dev)
            times = {arm.name: [] for arm in arms}
            for _ in range(a.runs):
                for arm in arms:
                    times[arm.name].append(time_arm(arm, a.iters, a.warmup))
            t0 = statistics.median(times[arms[0].name])
            rows = []
            for arm in arms:
                t = times[arm.name]
                med = statistics.median(t)
                rows.append(dict(arm=arm.name, ms_median=med, ms_min=min(t), ms_max=max(t), launches_per_step=arm.launches,
                                 minus_baseline_us=(med - t0) * 1e3, over_baseline=med / t0 - 1))
                launches = "torch ops only" if arm.launches is None else f"{arm.launches} launches/step"
                diff = "" if arm is arms[0] else (f"; vs {arms[0].name} {rows[-1]['minus_baseline_us']:+.1f} us/step, "
                                                  f"t/t0 - 1 = {rows[-1]['over_baseline']:+.4f}")
                print(f"B{B:<3d} {arm.name:16s}: {med:.3f} ms/step (min {min(t):.3f}, max {max(t):.3f}), {launches}{diff}",
                      flush=True)
            res["batches"].append(dict(batch=B, arms=rows))
            del arms, arm
            torch.cuda.empty_cache()
    finally:
        ops.set_pdl(False)
    print(f"after the runs: SM clock {smi('clocks.sm')}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
