#!/usr/bin/env python
"""Decode-step cost of GPTQ act-order weights (developer tool, runs on the GPU): Llama-3-8B INT4 g128, batch 32, context 2048,
CUDA graph + PDL, DecodeStep(act_order=False) and (act_order=True) timed alternately. act_order adds three gathers per layer
(x before qkv and w13, the attention output before o); w2's order is folded into w13 and costs nothing at run time.
Prints the card, its power limit and SM clock from the same run, then the median and range of ms/step of each arm."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200.decode_step import LLAMA3_8B, DecodeStep  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("act_order_step: needs a CUDA device")
    dev = torch.device("cuda:0")
    models = {}
    for ao in (False, True):
        m = DecodeStep(LLAMA3_8B, a.batch, a.ctx, dev, pdl=True, act_order=ao)
        m.capture()
        models[ao] = m
    launches = {ao: m.launches_per_step() for ao, m in models.items()}
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(a.runs):
        for ao in (False, True):
            times[ao].append(time_steps(models[ao], a.steps, a.warmup))
    print(f"{torch.cuda.get_device_name(0)}; power limit, SM clock, max SM clock: {smi('power.limit,clocks.sm,clocks.max.sm')}")
    print(f"{LLAMA3_8B.name} int4 g128 B{a.batch} ctx{a.ctx}, CUDA graph + PDL, {a.runs} runs x {a.steps} steps, alternating")
    for ao in (False, True):
        t = times[ao]
        print(f"act_order={str(ao):5s}: {statistics.median(t):.3f} ms/step (range {min(t):.3f}-{max(t):.3f}), "
              f"{launches[ao]} launches/step", flush=True)
    d = statistics.median(times[True]) / statistics.median(times[False]) - 1
    print(f"act-order cost: {100 * d:+.2f} % of the step")


if __name__ == "__main__":
    main()
