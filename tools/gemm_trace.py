#!/usr/bin/env python
"""Developer tool: per-k-block timeline (clock64) of CTA (0,0) of the weight-only GEMM (needs a B200_DEV=1 build)."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops
from rtp_llm_b200._lib import B200_FMT_INT4, B200_FMT_INT8

dev = torch.device("cuda:0")
fmt = {"int4": B200_FMT_INT4, "int8": B200_FMT_INT8}[sys.argv[1] if len(sys.argv) > 1 else "int4"]
B, K, N = 32, int(sys.argv[2]) if len(sys.argv) > 2 else 4096, int(sys.argv[3]) if len(sys.argv) > 3 else 28672
if fmt == B200_FMT_INT4:
    qp = torch.randint(0, 256, (K, N // 2), device=dev, dtype=torch.uint8)
    s = (torch.randn(K // 128, N, device=dev).abs() * 0.01 + 1e-3).half()
    w = ops.pack_w4(qp, s, s)
else:
    w = ops.pack_w8(torch.randint(-128, 128, (K, N), device=dev, dtype=torch.int8), torch.ones(N, device=dev).half())
x = torch.randn(B, K, device=dev).half()
ws = ops.gemm_workspace(B, [(K, N)], dev)
for _ in range(3):
    ops.wo_gemm(x, w, ws)
trace = torch.zeros(8 * 64 + 16 + 3 * 1024, dtype=torch.int64, device=dev)
trace[8 * 64 + 14] = 2**62
os.environ["B200_GEMM_TRACE_PTR"] = str(trace.data_ptr())
st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
st.record()
ops.wo_gemm(x, w, ws)
en.record()
torch.cuda.synchronize()
print("event-timed launch:", st.elapsed_time(en) * 1e3, "us")
os.environ.pop("B200_GEMM_TRACE_PTR")
ex = trace.cpu()[8 * 64:]
t = trace.cpu()[: 8 * 64].view(8, 64)
t0 = int(t[0, 0])
# slots written by the kernel (wo_gemm.cuh, B200_TRACE): 4 and 5 are unused
slots = {0: "w_issue", 1: "x_issue", 2: "dq_wfull", 3: "dq_math", 6: "mma_ready", 7: "mma_done"}
print("it  " + " ".join(f"{n:>11s}" for n in slots.values()))
for it in range(min(32, K // 128)):
    print(f"{it:2d}  " + " ".join(f"{int(t[r, it]) - t0 if int(t[r, it]) else -1:11d}" for r in slots))
print("all CTAs: earliest start -> latest end:", int(ex[15]) - int(ex[14]), "ns")
