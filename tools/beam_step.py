#!/usr/bin/env python
"""Cost of a beam-search decode step (developer tool, runs on the GPU): Llama-3-8B INT4 at ctx 2048, B requests x W beams
under CUDA graph + PDL, against the greedy step at B * W rows (the same row count), replayed in alternation, `--runs` times
each; each run times `--iters` graph replays with CUDA events. The two steps also differ in what they read: a request's beams
share the prompt's full pages (attention reads them once from HBM and then from L2), and the beam prompts are shorter. So
the fork is also timed on its own, as a graph of DecodeStep.fork() alone (its index ops and the copy of every row's partial
page in every layer), alternating with the two steps. A beam step advances its state, so every run starts again from the
prompt (upload_inputs, outside the timed window): the prompts hold ctx - max_new_tokens tokens (max_new_tokens = iters + 8),
the greedy step's ctx - 1. Writes JSON to --out."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, DecodeStep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--beam-width", type=int, default=4)
    ap.add_argument("--ngram", type=int, default=0)
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
    B, W = a.batch, a.beam_width
    steps = {"greedy": DecodeStep(LLAMA3_8B, B * W, a.ctx, dev, pdl=True),
             "beam": DecodeStep(LLAMA3_8B, B, a.ctx, dev, pdl=True, beam_width=W, no_repeat_ngram=a.ngram,
                                max_new_tokens=a.iters + 8)}
    for m in steps.values():
        m.capture()
    beam = steps["beam"]
    beam.replay()                                  # beam_out holds a real selection for the fork graph to replay
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        beam.fork()
    torch.cuda.current_stream().wait_stream(s)
    fork_graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(fork_graph):
        beam.fork()
    torch.cuda.synchronize()
    times = {k: [] for k in list(steps) + ["fork"]}
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k in times:
            replay = fork_graph.replay if k == "fork" else steps[k].replay
            beam.upload_inputs()
            for _ in range(3):
                replay()
            st.record()
            for _ in range(a.iters):
                replay()
            en.record()
            torch.cuda.synchronize()
            times[k].append(st.elapsed_time(en) / a.iters)
    beam.upload_inputs()
    ops.set_pdl(False)
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": power, "model": LLAMA3_8B.name, "ctx": a.ctx,
           "batch": B, "beam_width": W, "ngram": a.ngram, "runs": a.runs, "iters": a.iters}
    for k, t in times.items():
        t = sorted(t)
        res[k] = dict(ms_median=t[len(t) // 2], ms_min=t[0], ms_max=t[-1])
        print(f"{k:6s} ({'B%d x W%d' % (B, W) if k != 'greedy' else 'B%d' % (B * W)}): {t[len(t) // 2]:7.3f} ms/step "
              f"(min {t[0]:.3f}, max {t[-1]:.3f})", flush=True)
    res["beam_minus_greedy_ms"] = res["beam"]["ms_median"] - res["greedy"]["ms_median"]
    print(f"beam - greedy: {res['beam_minus_greedy_ms'] * 1e3:.1f} us/step", flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
