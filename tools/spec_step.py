#!/usr/bin/env python
"""Cost of a speculative-token verification step (developer tool, runs on the GPU): Llama-3-8B INT4 at ctx 2048 (or
Llama-3.1-8B with its Llama3 rope scaling, --model llama31), one
DecodeStep per (batch, q_len) with batch * q_len <= 128, CUDA graph + PDL. The q_len variants of a batch are replayed in
alternation, `--runs` times each, and each run times `--iters` graph replays with CUDA events. Prints ms per step and the break-even
number of accepted drafts per step, t(q_len) / t(1) - 1: a verification step of q_len tokens pays off when it accepts more
drafts than that on average. Writes the JSON result to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, LLAMA31_8B, DecodeStep  # noqa: E402

MODELS = {"llama3": LLAMA3_8B, "llama31": LLAMA31_8B}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS), default="llama3")
    ap.add_argument("--batches", default="8,16,32")
    ap.add_argument("--q-lens", default="1,2,4")
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    ops.device_check(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(0), "| name, power limit:", power or "unknown", flush=True)
    cfgs = [(B, n) for B in map(int, a.batches.split(",")) for n in map(int, a.q_lens.split(",")) if B * n <= 128]
    times = {c: [] for c in cfgs}
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for B in sorted({c[0] for c in cfgs}):             # one batch at a time: its q_len variants are held together
        steps = {}
        for c in [c for c in cfgs if c[0] == B]:
            m = DecodeStep(MODELS[a.model], B, a.ctx, dev, pdl=True, q_len=c[1])
            m.capture()
            steps[c] = m
        for _ in range(a.runs):
            for c, m in steps.items():                  # alternate the q_len variants within every run
                for _ in range(3):
                    m.replay()
                st.record()
                for _ in range(a.iters):
                    m.replay()
                en.record()
                torch.cuda.synchronize()
                times[c].append(st.elapsed_time(en) / a.iters)
        del steps, m
        torch.cuda.empty_cache()
    ops.set_pdl(False)
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": power, "model": MODELS[a.model].name, "ctx": a.ctx, "runs": a.runs, "rows": []}
    for B, n in cfgs:
        t = sorted(times[(B, n)])
        med = t[len(t) // 2]
        base = sorted(times[(B, 1)])[len(times[(B, 1)]) // 2] if (B, 1) in times else None
        be = (med / base - 1.0) if base else None
        res["rows"].append(dict(batch=B, q_len=n, ms_median=med, ms_min=t[0], ms_max=t[-1], break_even_accepted=be))
        print(f"B{B:3d} q_len {n}: {med:7.3f} ms/step (min {t[0]:.3f}, max {t[-1]:.3f})"
              + (f"  break-even accepted drafts/step {be:.2f}" if be is not None else ""), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
