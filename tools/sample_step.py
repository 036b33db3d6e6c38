#!/usr/bin/env python
"""Cost of a sampled decode step (developer tool, runs on the GPU): Llama-3-8B INT4 at ctx 2048 under CUDA graph + PDL, the
sampling mode (temperature 0.8, top-k 50, top-p 0.9, repetition 1.1, the drawn token's log-prob and the top 5) against the
greedy step at the same batch, replayed in alternation, `--runs` times each; each run times `--iters` graph replays with CUDA
events. A sampled step advances its state, so every run starts again from the prompt (upload_inputs, outside the timed
window): its prompts hold ctx - max_new_tokens tokens (max_new_tokens = iters + 8), the greedy step's ctx - 1. Writes JSON
to --out."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, DecodeStep, SamplingParams  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    ops.device_check(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(0), "| name, power limit:", power or "unknown", flush=True)
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": power, "model": LLAMA3_8B.name, "ctx": a.ctx,
           "runs": a.runs, "iters": a.iters}
    sp = SamplingParams(temperature=0.8, top_k=50, top_p=0.9, repetition=1.1, seed=1)
    for B in a.batch:
        steps = {"greedy": DecodeStep(LLAMA3_8B, B, a.ctx, dev, pdl=True),
                 "sampled": DecodeStep(LLAMA3_8B, B, a.ctx, dev, pdl=True, sampling=sp, logprobs=5, max_new_tokens=a.iters + 8)}
        launches = {k: m.launches_per_step() for k, m in steps.items()}
        for m in steps.values():
            m.upload_inputs()
            m.capture()
        times = {k: [] for k in steps}
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.runs):
            for k, m in steps.items():
                m.upload_inputs()
                for _ in range(3):
                    m.replay()
                m.upload_inputs()
                torch.cuda.synchronize()
                st.record()
                for _ in range(a.iters):
                    m.replay()
                en.record()
                torch.cuda.synchronize()
                times[k].append(st.elapsed_time(en) / a.iters)
        r = {"launches_per_step": launches}
        for k, t in times.items():
            t = sorted(t)
            r[k] = dict(ms_median=t[len(t) // 2], ms_min=t[0], ms_max=t[-1])
            print(f"B{B} {k:7s}: {t[len(t) // 2]:7.3f} ms/step (min {t[0]:.3f}, max {t[-1]:.3f}), {launches[k]} native launches",
                  flush=True)
        r["sampled_minus_greedy_ms"] = r["sampled"]["ms_median"] - r["greedy"]["ms_median"]
        print(f"B{B} sampled - greedy: {r['sampled_minus_greedy_ms'] * 1e3:.1f} us/step", flush=True)
        res[f"B{B}"] = r
        del steps
        torch.cuda.empty_cache()
    ops.set_pdl(False)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
