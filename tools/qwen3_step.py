#!/usr/bin/env python
"""Decode-step A/B of Qwen3's QK-norm (developer tool, runs on the GPU): Qwen3-8B INT4 g128, context 2048, CUDA graph + PDL,
at batch 8, 16 and 32. The step as built (QK-RMSNorm inside the rope launch, b200_qk_norm_rope_append) is timed alternately
against TwoLaunchStep below, which runs b200_qk_rmsnorm in place on qkv and then the plain rope launch: one launch more per
layer, the same logits. Prints the card, its power limit and SM clock from the same run, then per batch the median and range of
ms/step of each arm and its launches per step."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops, rope  # noqa: E402
from rtp_llm_b200.decode_step import QWEN3_8B, DecodeStep  # noqa: E402


class TwoLaunchStep(DecodeStep):
    """The composition the fused launch replaces: qk_rmsnorm in place on qkv, then rope.rope_append without QK-norm."""

    def _rope_append(self, L):
        ops.qk_rmsnorm(self.qkv, L["q_norm"], L["k_norm"], self.Hq, self.Hkv, self.D, self.cfg.eps)
        rope.rope_append(self.rope_spec, self.qkv, L["kv"], self.page_list, self.seq_lens, self.Hq, q_out=self.q, q_len=self.q_len)


def smi(fields: str) -> str:
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip() or "unknown"


def time_steps(model: DecodeStep, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        model.replay()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(steps):
        model.replay()
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qwen3_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    arms = {"fused": DecodeStep, "norm + rope": TwoLaunchStep}
    print(f"{torch.cuda.get_device_name(0)}; power limit, SM clock, max SM clock: {smi('power.limit,clocks.sm,clocks.max.sm')}")
    print(f"{QWEN3_8B.name} int4 g128 ctx{a.ctx}, CUDA graph + PDL, {a.runs} runs x {a.steps} steps, arms alternating", flush=True)
    for B in a.batch:
        models = {}
        for name, cls in arms.items():
            m = cls(QWEN3_8B, B, a.ctx, dev, pdl=True)
            m.capture()
            models[name] = m
        launches = {name: m.launches_per_step() for name, m in models.items()}
        torch.cuda.synchronize()
        same = torch.equal(models["fused"].logits, models["norm + rope"].logits)
        times = {name: [] for name in arms}
        for _ in range(a.runs):
            for name in arms:
                times[name].append(time_steps(models[name], a.steps, a.warmup))
        for name in arms:
            t = times[name]
            print(f"B{B:<3d} {name:12s}: {statistics.median(t):.3f} ms/step (range {min(t):.3f}-{max(t):.3f}), "
                  f"{launches[name]} launches/step", flush=True)
        d = statistics.median(times["fused"]) / statistics.median(times["norm + rope"]) - 1
        print(f"B{B:<3d} fused vs norm + rope: {100 * d:+.2f} % of the step; logits bit-identical: {same}", flush=True)
        del models
        torch.cuda.empty_cache()
    print(f"after the runs: SM clock {smi('clocks.sm')}")


if __name__ == "__main__":
    main()
