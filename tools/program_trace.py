#!/usr/bin/env python
"""Per-op timeline of a decode program (developer tool, run under gpurun): every CTA's dq role stamps %globaltimer at op
entry / exit into a trace buffer (b200_program_set_trace). Prints, per op of one layer: when the first CTA entered, when the
last CTA left, the busiest CTA's time inside the op, and the gap to the previous op (barrier + dependency wait)."""
import dataclasses
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, QWEN2_72B, DecodeStep  # noqa: E402

dev = torch.device("cuda:0")


def main():
    layers = int(os.environ.get("LAYERS", "4"))
    batch = int(os.environ.get("BATCH", "32"))
    ctx = int(os.environ.get("CTX", "2048"))
    quant = os.environ.get("QUANT", "int4")
    pdl = int(os.environ.get("PDL", "1"))
    cfg = dataclasses.replace(LLAMA3_8B, layers=layers, quant=quant)
    m = DecodeStep(cfg, batch, ctx, dev, pdl=bool(pdl))
    m.build_program()
    G = int(os.environ.get("GRID", 2 * torch.cuda.get_device_properties(0).multi_processor_count))
    nops = m.prog.num_ops
    FTS, FTB = 8, 48
    trace = torch.zeros(nops * G * 2 + nops * FTS * FTB, dtype=torch.int64, device=dev)
    m.prog.set_trace(trace)
    for _ in range(3):
        m.run()
    torch.cuda.synchronize()
    trace.zero_()
    m.run()
    torch.cuda.synchronize()
    raw = trace.cpu().numpy()
    t = raw[: nops * G * 2].reshape(nops, G, 2).astype(np.float64)
    ft = raw[nops * G * 2:].reshape(nops, FTS, FTB).astype(np.float64)
    names = []
    # op order recorded by DecodeStep.step_core
    names += ["blocktable", "embed"]
    for l in range(layers):
        names += ["norm1", "qkv", "rope", "o", "norm2", "w13", "w2"]
    names += ["normf"]
    assert len(names) == nops, (len(names), nops)
    t0 = t[t > 0].min()
    print(f"program: {nops} fused ops, {m.prog.num_launches} launches; G={G}; times in us relative to the first stamp")
    print(f"{'op':>3} {'name':>10} {'first_in':>9} {'last_in':>9} {'first_out':>9} {'last_out':>9} {'span':>7} {'max_cta':>8} {'med_cta':>8} {'gap_prev':>8}")
    prev_out = None
    for i in range(nops):
        s, e = t[i, :, 0], t[i, :, 1]
        ok = (s > 0) & (e > 0)
        if not ok.any():
            print(f"{i:3d} {names[i]:>10} (no stamps)")
            continue
        s, e = (s[ok] - t0) / 1e3, (e[ok] - t0) / 1e3
        d = e - s
        gap = (s.min() - prev_out) if prev_out is not None else 0.0
        print(f"{i:3d} {names[i]:>10} {s.min():9.2f} {s.max():9.2f} {e.min():9.2f} {e.max():9.2f} {e.max() - s.min():7.2f} {d.max():8.2f} {np.median(d):8.2f} {gap:8.2f}")
        prev_out = e.max()
    show = [i for i, n in enumerate(names) if n in ("w13", "o")][2:4]
    fine(ft, names, show)




def fine(ft, names, ops_to_show):
    # slots written by decode_program.cuh (B200_FT): 3 and 4 are unused; slot 7 holds the epilogue stamps
    slots = {0: "w_issue", 1: "x_issue", 2: "dq_wfull", 5: "mma_ready", 6: "mma_done"}
    for i in ops_to_show:
        f = ft[i]
        base = f[f > 0].min() if (f > 0).any() else 0
        print(f"--- fine timeline of CTA 0, op {i} ({names[i]}): cycles since the op's first stamp; dq columns = warpgroup 0")
        print(" blk " + " ".join(f"{s:>10}" for s in slots.values()))
        for b in range(48):
            if not any(f[sl, b] > 0 for sl in slots):
                continue
            print(f"{b:4d} " + " ".join(f"{(f[sl, b] - base) if f[sl, b] > 0 else -1:10.0f}" for sl in slots))
        ep = f[7]
        print(" epilogues (segment: begin, done): " + ", ".join(
            f"[{ep[2*c]-base:.0f}, {ep[16+c]-base:.0f}]" for c in range(8) if ep[2*c] > 0))

if __name__ == "__main__":
    main()
