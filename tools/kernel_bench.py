#!/usr/bin/env python
"""Per-kernel timing at the BASELINE shapes (developer tool, runs on the GPU). CUDA events on the launching stream,
warm-up, inputs rotated through > L2-size working sets so nothing is served from the H100's 50 MB L2."""
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_F16, B200_FMT_INT4, B200_FMT_INT8  # noqa: E402

dev = torch.device("cuda:0")
PEAK = 3350.0          # H100 SXM data-sheet HBM3 bandwidth (GB/s); a measured peak replaces it when present
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:  # noqa: BLE001
    pass


def timeit(fn, n_rot, iters=20, warm=3):
    """Average device time per call with the calls replayed from a CUDA graph (no CPU launch overhead in the number)."""
    calls = max(n_rot, 8)
    for i in range(calls):
        fn(i % n_rot)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(calls):
            fn(i % n_rot)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(calls):
            fn(i % n_rot)
    for _ in range(warm):
        g.replay()
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.record()
    for _ in range(iters):
        g.replay()
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / (iters * calls) * 1e3  # us


def bench_attn(B, Hq, Hkv, S, T=64, nrot=3, env=None):
    for k, v in (env or {}).items():
        os.environ[k] = str(v)
    M = math.ceil(S / T)
    P = B * M + 1
    pools = [torch.randn(P, 2, Hkv, T, 128, device=dev).half() for _ in range(nrot)]
    q = torch.randn(B, Hq, 128, device=dev).half()
    bid = (torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M)
    pl = ops.convert_block_table(bid)
    seq = torch.full((B,), S - 1, dtype=torch.int32, device=dev)
    ws = ops.attn_workspace(B, Hq, Hkv, S, dev)
    out = torch.empty(B, Hq * 128, device=dev).half()
    us = timeit(lambda i: ops.paged_decode_attn(q, pools[i], pl, seq, S, ws, out=out), nrot)
    byt = 2 * B * S * Hkv * 128 * 2
    for k in (env or {}):
        os.environ.pop(k, None)
    print(f"attn B{B} Hq{Hq} Hkv{Hkv} S{S} {env or ''}: {us:8.1f} us  {byt / us / 1e3:7.0f} GB/s  frac={byt / us / 1e3 / PEAK:.3f}", flush=True)
    return us


def bench_attn_multi(B, Hq, Hkv, S, q_len, T=64, nrot=3):
    """b200_paged_decode_attn_multi with q_len query tokens per sequence (group * q_len query rows per kv head); the K/V bytes
    are those of plain decode, 2*B*S*Hkv*D*2 with S the cached length the last query sees."""
    M = math.ceil(S / T)
    P = B * M + 1
    pools = [torch.randn(P, 2, Hkv, T, 128, device=dev).half() for _ in range(nrot)]
    q = torch.randn(B, q_len, Hq, 128, device=dev).half()
    bid = (torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M)
    pl = ops.convert_block_table(bid)
    seq = torch.full((B,), S - q_len, dtype=torch.int32, device=dev)
    ws = ops.attn_workspace(B * q_len, Hq, Hkv, S, dev)
    out = torch.empty(B, q_len, Hq * 128, device=dev).half()
    us = timeit(lambda i: ops.paged_decode_attn_multi(q, pools[i], pl, seq, S, ws, out=out), nrot)
    byt = 2 * B * S * Hkv * 128 * 2
    print(f"attn-multi B{B} Hq{Hq} Hkv{Hkv} S{S} q_len {q_len} (rows {Hq // Hkv * q_len}): {us:8.1f} us  {byt / us / 1e3:7.0f} GB/s  "
          f"frac={byt / us / 1e3 / PEAK:.3f}", flush=True)
    return us


def bench_attn_tree(B, Hq, Hkv, S, q_len, kind, T=64, nrot=3, runs=3):
    """b200_paged_decode_attn_tree against b200_paged_decode_attn_multi on the same rows and tables, alternating; kind: the
    tree's shape (chain, star or binary). The mask only touches the slices that reach the new tokens."""
    M = math.ceil(S / T)
    P = B * M + 1
    pools = [torch.randn(P, 2, Hkv, T, 128, device=dev).half() for _ in range(nrot)]
    q = torch.randn(B, q_len, Hq, 128, device=dev).half()
    bid = (torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M)
    pl = ops.convert_block_table(bid)
    seq = torch.full((B,), S - q_len, dtype=torch.int32, device=dev)
    par = [-1] + [{"chain": j - 1, "star": 0, "binary": (j - 1) // 2}[kind] for j in range(1, q_len)]
    parents = torch.tensor([par] * B, dtype=torch.int32, device=dev)
    ws = ops.attn_workspace(B * q_len, Hq, Hkv, S, dev)
    out = torch.empty(B, q_len, Hq * 128, device=dev).half()
    arms = {"multi": lambda i: ops.paged_decode_attn_multi(q, pools[i], pl, seq, S, ws, out=out),
            "tree": lambda i: ops.paged_decode_attn_tree(q, pools[i], pl, seq, parents, S, ws, out=out)}
    t = {k: [] for k in arms}
    for _ in range(runs):
        for k, fn in arms.items():
            t[k].append(timeit(fn, nrot))
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    print(f"attn-tree B{B} Hq{Hq} Hkv{Hkv} S{S} q_len {q_len} {kind} median: multi {med['multi']:.1f} us, tree {med['tree']:.1f} us "
          f"({med['tree'] / med['multi']:.3f}x)", flush=True)
    return med


def bench_tree_verify(B, n, sampling, V=128256, nrot=4):
    """b200_spec_verify_tree on binary trees of n nodes, greedy or sampled (target rows of temperature-0.25 softmaxes)."""
    par = torch.tensor([[-1] + [(j - 1) // 2 for j in range(1, n)]] * B, dtype=torch.int32, device=dev)
    ids = torch.randint(0, V, (B, n), dtype=torch.int32, device=dev)
    toks = [ids.gather(1, par.clamp(min=0).long()).to(torch.int32).contiguous() for _ in range(nrot)]
    probs = [torch.softmax(torch.randn(B, n, V, device=dev) / 0.25, dim=-1) for _ in range(nrot)] if sampling else None
    u = torch.rand(B, n, device=dev)
    if sampling:
        fn = lambda i: ops.spec_verify_tree(par, toks[i], target_probs=probs[i], uniform=u)
    else:
        fn = lambda i: ops.spec_verify_tree(par, toks[i], target_ids=ids)
    us = timeit(fn, nrot)
    print(f"tree-verify B{B} n{n} {'sampled' if sampling else 'greedy'}: {us:.1f} us", flush=True)
    return us


def bench_kv_compact(B, layers=32, Hkv=8, T=64, n=8, S=2048, nrot=2):
    """b200_kv_compact_path over the Llama-3-8B cache (32 layers, Hkv 8, D 128) with a path that moves every depth."""
    M = math.ceil((S + n) / T)
    P = B * M + 1
    caches = [torch.randn(P, 2, Hkv, T, 128, device=dev).half() for _ in range(layers)]
    pl = ops.convert_block_table((torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M))
    seq = torch.full((B,), S, dtype=torch.int32, device=dev)
    a = n // 2
    path = torch.tensor([[0] + [d + 1 for d in range(1, a + 1)] + [-1] * (n - a - 1)] * B, dtype=torch.int32, device=dev)
    acc = torch.full((B,), a, dtype=torch.int32, device=dev)
    us = timeit(lambda i: ops.kv_compact_path(caches, pl, seq, path, acc), nrot)
    byt = 2 * 2 * B * layers * Hkv * a * 128 * 2
    print(f"kv-compact B{B} layers {layers} accepted {a}: {us:.2f} us ({byt / 1e6:.2f} MB moved)", flush=True)
    return us


def bench_attn_beam(B, W, Hq, Hkv, S=2048, T=64, private=28, nrot=3, runs=3):
    """b200_paged_decode_attn_beam against b200_paged_decode_attn on the same B * W rows and the same page tables, whose beams
    share the full pages of the first S - private tokens and own the pages after them (the beam step's tables), the arms
    alternating; and the beam kernel with shared_lengths 0 on those tables: what the expansion into one stage per beam costs
    by itself. GB/s is distinct bytes over kernel time, the K/V bytes that differ between rows (a request's shared pages
    once): HBM traffic of the beam arm, not of the per-row arm, which reads the shared pages once per beam from HBM or L2."""
    M, R = math.ceil(S / T), B * W
    shared_pages = (S - private) // T
    P = B * shared_pages + R * (M - shared_pages) + 1
    pools = [torch.randn(P, 2, Hkv, T, 128, device=dev).half() for _ in range(nrot)]
    q = torch.randn(B, W, Hq, 128, device=dev).half()
    ids = iter((torch.randperm(P - 1) + 1).tolist())
    bid = torch.zeros(R, M, dtype=torch.int32)
    for b in range(B):
        common = [next(ids) for _ in range(shared_pages)]
        for i in range(W):
            bid[b * W + i] = torch.tensor(common + [next(ids) for _ in range(M - shared_pages)], dtype=torch.int32)
    pl = ops.convert_block_table(bid.to(dev))
    seq = torch.full((R,), S - 1, dtype=torch.int32, device=dev)
    shared = torch.full((B,), shared_pages * T, dtype=torch.int32, device=dev)
    zero = torch.zeros_like(shared)
    ws = ops.attn_workspace(R, Hq, Hkv, S, dev)
    out = torch.empty(B, W, Hq * 128, device=dev).half()
    arms = {"per row": lambda i: ops.paged_decode_attn(q.view(R, Hq, 128), pools[i], pl, seq, S, ws, out=out.view(R, -1)),
            "beam": lambda i: ops.paged_decode_attn_beam(q, pools[i], pl, seq, shared, S, ws, out=out),
            "beam shared 0": lambda i: ops.paged_decode_attn_beam(q, pools[i], pl, seq, zero, S, ws, out=out)}
    t = {k: [] for k in arms}
    for _ in range(runs):
        for k, fn in arms.items():
            t[k].append(timeit(fn, nrot))
    byt = 2 * (B * shared_pages * T + R * (S - shared_pages * T)) * Hkv * 128 * 2
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    print(f"attn-beam B{B} W{W} Hq{Hq} Hkv{Hkv} S{S} (rows {Hq // Hkv * W}, {byt / 1e6:.0f} MB distinct K/V): " + ", ".join(
        f"{k} {med[k]:.1f} us (min {min(t[k]):.1f}, max {max(t[k]):.1f}; distinct bytes over kernel time {byt / med[k] / 1e3:.0f} GB/s)"
        for k in arms) + f"; beam / per row = {med['beam'] / med['per row']:.2f}", flush=True)
    return med


def bench_beam(B, W, V=128256, ngram=0, hist=2048, nrot=8):
    """b200_beam_search_step on fp16 logits [B*W, V] (rotated through nrot sets, > L2), preceded by b200_ban_repeat_ngram
    over `hist` history tokens per row when ngram > 0."""
    rows = B * W
    g = torch.Generator(device=dev).manual_seed(1)
    xs = [(torch.randn(rows, V, generator=g, device=dev) * 3).half() for _ in range(nrot)]
    cum = -torch.rand(B, W, generator=g, device=dev)
    ws = ops.beam_search_workspace(B, W, V, dev)
    out = ops.beam_search_step(xs[0], cum, W, workspace=ws)
    h = torch.randint(0, 64, (rows, hist), generator=g, device=dev, dtype=torch.int32)
    hl = torch.full((rows,), hist, dtype=torch.int32, device=dev)
    ng = torch.full((rows,), ngram, dtype=torch.int32, device=dev)

    def fn(i):
        if ngram > 0:
            ops.ban_repeat_ngram(xs[i], h, hl, ng)
        ops.beam_search_step(xs[i], cum, W, workspace=ws, out=out)
    us = timeit(fn, nrot)
    print(f"beam B{B} W{W} V{V}" + (f" + ban n{ngram} over {hist}" if ngram else "") + f": {us:8.1f} us", flush=True)
    return us


def bench_beam_hyps(B, W, max_len, nrot=8):
    """b200_beam_hypotheses_update and b200_beam_hypotheses_finalize (n = W), each timed on its own. The update sees a
    non-EOS best candidate of score 0 (so no request is ever done: every hypothesis scores below it), then EOS at ranks
    1..2W-1 with fresh scores (rotated through nrot candidate sets), parent paths of max_len - 1 tokens, length penalty 1. "steady" keeps the state across calls: the sets are
    full and a candidate enters only when it beats the worst. "empty" zeroes the state before every call (the memset is in the
    time), so every call inserts W - 1 hypotheses and copies their paths of max_len tokens. Finalize merges W live beams of max_len - 1
    tokens into the full sets and writes n = W."""
    g = torch.Generator(device=dev).manual_seed(4)
    K, R = 2 * W, B * W
    cands = []
    for _ in range(nrot):
        score = -torch.rand(B, K, generator=g, device=dev).mul_(8.0).sort(dim=1).values
        score[:, 0] = 0.0
        token = torch.full((B, K), 2, dtype=torch.int32, device=dev)
        token[:, 0] = 3
        cands.append(dict(cand_token=token,
                          cand_parent=torch.randint(0, W, (B, K), generator=g, device=dev, dtype=torch.int32), cand_score=score))
    hist = torch.randint(0, 128256, (R, max_len), generator=g, device=dev, dtype=torch.int32)
    hl = torch.full((R,), max_len, dtype=torch.int32, device=dev)
    lp = torch.ones(B, device=dev)
    es = torch.full((B,), 2, dtype=torch.int32, device=dev)
    state = ops.beam_hypotheses_state(B, W, max_len, dev)
    done = torch.zeros(B, dtype=torch.int32, device=dev)
    cum = -torch.rand(B, W, generator=g, device=dev)
    out = ops.beam_hypotheses_finalize(state, done, cum, hist, hl, W, max_len, lp, gen_start=1)

    def update(i, empty):
        if empty:
            state.zero_()
        ops.beam_hypotheses_update(cands[i], hist, hl, 2, lp, es, state, done, max_len, gen_start=1)
    empty = timeit(lambda i: update(i, True), nrot)
    up = timeit(lambda i: update(i, False), nrot)
    fin = timeit(lambda i: ops.beam_hypotheses_finalize(state, done, cum, hist, hl, W, max_len, lp, gen_start=1, out=out), nrot)
    assert int(done.sum()) == 0
    print(f"beam-hyps B{B} W{W} max_len {max_len}: update steady {up:7.2f} us, empty (+ memset) {empty:7.2f} us, "
          f"finalize {fin:7.2f} us", flush=True)
    return up, empty, fin


def bench_logprobs(B, top_n, V=128256, nrot=8):
    """b200_token_logprobs on fp16 logits [B, V] (rotated through nrot sets, > L2): the drawn token's log-prob and the top_n."""
    g = torch.Generator(device=dev).manual_seed(2)
    xs = [(torch.randn(B, V, generator=g, device=dev) * 3).half() for _ in range(nrot)]
    tok = torch.randint(0, V, (B,), generator=g, device=dev, dtype=torch.int32)
    ws = ops.token_logprobs_workspace(B, V, top_n, dev)
    out = ops.token_logprobs(xs[0], top_n, tokens=tok, workspace=ws)
    us = timeit(lambda i: ops.token_logprobs(xs[i], top_n, tokens=tok, workspace=ws, out=out), nrot)
    print(f"logprobs B{B} V{V} top_n {top_n}: {us:8.1f} us  {B * V * 2 / us / 1e3:7.0f} GB/s", flush=True)
    return us


def bench_sample(B, top_k, top_p, V=128256, nrot=4, copy_only=False, min_p=None):
    """b200_sample on fp32 logits [B, V] at temperature 0.8 with every row's top_k / top_p (and min_p when given). The op works
    in place, so each call first copies fresh logits into its buffer (rotated through nrot sources); copy_only times that copy
    alone."""
    g = torch.Generator(device=dev).manual_seed(3)
    src = [torch.randn(B, V, generator=g, device=dev) * 3 for _ in range(nrot)]
    x = torch.empty(B, V, device=dev)
    k = torch.full((B,), top_k, dtype=torch.int32, device=dev)
    p = torch.full((B,), top_p, device=dev)
    t = torch.full((B,), 0.8, device=dev)
    u = torch.rand(B, generator=g, device=dev)
    out = dict(token=torch.empty(B, dtype=torch.int32, device=dev), token_prob=torch.empty(B, device=dev))
    mp = None if min_p is None else torch.full((B,), min_p, device=dev)

    def fn(i):
        x.copy_(src[i])
        if not copy_only:
            ops.sample(x, k, p, u, temperature=t, out=out, min_p=mp)
    us = timeit(fn, nrot)
    what = "copy alone" if copy_only else f"copy + sample top_k {top_k} top_p {top_p}" + ("" if min_p is None else f" min_p {min_p}")
    print(f"sample B{B} V{V} {what}: {us:8.1f} us", flush=True)
    return us


def bench_constrain(rows, V, mask, bias, dtype=torch.float16):
    """b200_constrain_logits on logits [rows, V] (rotated through > L2 of sets) with an all-ones ("ones"), a 50 % random
    ("half") or a single-token ("single") mask, and 0 or `bias` entries per row on random tokens. Bytes = the mask words read,
    the masked logits written, and per bias entry its id and value read and its logit read and written when it is allowed."""
    g = torch.Generator(device=dev).manual_seed(4)
    es = torch.finfo(dtype).bits // 8
    nrot = max(2, int(200e6 // (rows * V * es)) + 1)
    xs = [torch.randn(rows, V, generator=g, device=dev).to(dtype) for _ in range(nrot)]
    words = (V + 31) // 32
    if mask == "ones":
        ok = torch.ones(rows, words * 32, dtype=torch.bool, device=dev)
    elif mask == "half":
        ok = torch.rand(rows, words * 32, generator=g, device=dev) < 0.5
    else:
        ok = torch.zeros(rows, words * 32, dtype=torch.bool, device=dev)
        ok[torch.arange(rows, device=dev), torch.randint(0, V, (rows,), generator=g, device=dev)] = True
    ok[:, V:] = False
    m = (ok.view(rows, words, 32).to(torch.int64) << torch.arange(32, device=dev)).sum(-1)
    m = torch.where(m >= 2 ** 31, m - 2 ** 32, m).to(torch.int32)
    lb = None
    byt = rows * words * 4 + int((~ok[:, :V]).sum()) * es
    if bias:
        ids = torch.stack([torch.randperm(V, generator=g, device=dev)[:bias] for _ in range(rows)])
        lb = (torch.arange(rows + 1, dtype=torch.int32, device=dev) * bias, ids.to(torch.int32).view(-1),
              torch.randn(rows * bias, generator=g, device=dev))
        byt += rows * bias * 8 + int(ok.gather(1, ids).sum()) * 2 * es
    us = timeit(lambda i: ops.constrain_logits(xs[i], m, lb), nrot)
    print(f"constrain {str(dtype)[6:]} rows {rows} V{V} mask {mask:6s} bias {bias:3d}/row: {us:7.2f} us  {byt / 1e6:7.3f} MB  "
          f"{byt / us / 1e3:6.0f} GB/s", flush=True)
    return us


def bench_rope(kind, B, Hq, Hkv, q_len, S=2048, T=64, D=128, nrot=4):
    """RoPE + K/V append of q_len tokens per sequence at cached length S - q_len: b200_rope_append(_multi) ("base") against
    b200_rope_append_ex(_multi) with the Llama3 in-kernel formula ("llama3") or the Yarn cos/sin table ("yarn table").
    Bytes = qkv read + q written + K/V written (+ the table rows read)."""
    from rtp_llm_b200 import rope
    M = math.ceil(S / T)
    P = B * M + 1
    pools = [torch.zeros(P, 2, Hkv, T, D, device=dev).half() for _ in range(nrot)]
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, device=dev).half()
    q = torch.empty(B * q_len, Hq * D, device=dev).half()
    pl = ops.convert_block_table((torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M))
    seq = torch.full((B,), S - q_len, dtype=torch.int32, device=dev)
    spec = {"llama3": rope.RopeSpec(style=rope.LLAMA3, dim=D, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192),
            "yarn table": rope.RopeSpec(style=rope.YARN, dim=D, base=1000000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=32768,
                                        mscale=1.14)}.get(kind)
    if spec is None:
        fn = lambda i: ops.rope_append(qkv, pools[i], pl, seq, Hq, 500000.0, q_out=q, q_len=q_len)
        tbytes = 0
    else:
        rc, table = rope.c_config(spec), rope.table(spec, dev)
        fn = lambda i: ops.rope_append_ex(qkv, pools[i], pl, seq, Hq, rc, q_out=q, cos_sin_cache=table, q_len=q_len)
        tbytes = B * q_len * D * 4 if table is not None else 0
    us = timeit(fn, nrot)
    byt = B * q_len * ((Hq + 2 * Hkv) * D * 2 + (Hq + 2 * Hkv) * D * 2) + tbytes
    print(f"rope {kind:10s} B{B} Hq{Hq} Hkv{Hkv} D{D} q_len {q_len}: {us:7.2f} us  {byt / us / 1e3:7.0f} GB/s", flush=True)
    return us


def bench_qknorm_rope(kind, fused, B, Hq, Hkv, q_len, S=2048, T=64, D=128, nrot=4):
    """Qwen3's QK-RMSNorm + RoPE + K/V append of q_len tokens per sequence at cached length S - q_len, plain Base at base 1e6
    ("base") or Qwen3's Yarn cos/sin table ("yarn table"): the one-launch b200_qk_norm_rope_append(_ex) (fused) against
    b200_qk_rmsnorm in place on qkv followed by b200_rope_append(_ex) (two launches). Bytes = those of the fused kernel, qkv
    read + q and K/V written (+ the table rows); the composition moves the q and k heads once more."""
    from rtp_llm_b200 import rope
    M = math.ceil(S / T)
    P = B * M + 1
    pools = [torch.zeros(P, 2, Hkv, T, D, device=dev).half() for _ in range(nrot)]
    qkv = torch.randn(B * q_len, (Hq + 2 * Hkv) * D, device=dev).half()
    q = torch.empty(B * q_len, Hq * D, device=dev).half()
    qg, kg = (1 + 0.1 * torch.randn(D, device=dev)).half(), (1 + 0.1 * torch.randn(D, device=dev)).half()
    pl = ops.convert_block_table((torch.randperm(P - 1, device=dev).to(torch.int32) + 1).reshape(B, M))
    seq = torch.full((B,), S - q_len, dtype=torch.int32, device=dev)
    spec = (rope.RopeSpec(dim=D, base=1000000.0) if kind == "base" else
            rope.RopeSpec(style=rope.YARN, dim=D, base=1000000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=32768, mscale=1.14))
    rope.table(spec, dev)

    def fn(i):
        if fused:
            rope.rope_append(spec, qkv, pools[i], pl, seq, Hq, q_out=q, q_len=q_len, qk_norm=(qg, kg, 1e-6))
        else:
            ops.qk_rmsnorm(qkv, qg, kg, Hq, Hkv, D, 1e-6)
            rope.rope_append(spec, qkv, pools[i], pl, seq, Hq, q_out=q, q_len=q_len)
    us = timeit(fn, nrot)
    byt = B * q_len * 2 * (Hq + 2 * Hkv) * D * 2 + (B * q_len * D * 4 if kind != "base" else 0)
    print(f"qknorm-rope {kind:10s} {'fused' if fused else 'norm + rope':11s} B{B} Hq{Hq} Hkv{Hkv} D{D} q_len {q_len}: {us:7.2f} us  "
          f"{byt / us / 1e3:7.0f} GB/s", flush=True)
    return us


def bench_permute(B, K, nrot=4):
    """b200_permute_cols on [B, K] fp16; bytes = the row read and written, plus the perm."""
    xs = [torch.randn(B, K, device=dev).half() for _ in range(nrot)]
    perm = torch.randperm(K, device=dev).to(torch.int32)
    y = torch.empty(B, K, device=dev).half()
    us = timeit(lambda i: ops.permute_cols(xs[i], perm, out=y), nrot)
    byt = 2 * 2 * B * K + 4 * K
    print(f"permute_cols B{B} K{K}: {us:8.2f} us  {byt / us / 1e3:7.0f} GB/s", flush=True)
    return us


def bench_gemm(fmt, B, K, N, env=None, pdl=False, group=128, act_order=False):
    """group: quantisation group of INT4 weights (128, 64, 32); bytes count the scale and zero*scale of every group.
    act_order: the weight carries a row order (GPTQ act-order), so each call is the x gather plus the GEMM."""
    for k, v in (env or {}).items():
        os.environ[k] = str(v)
    nm = {B200_FMT_F16: "f16", B200_FMT_INT8: "int8", B200_FMT_INT4: f"int4 g{group}"}[fmt]
    wbytes = {B200_FMT_F16: 2 * K * N, B200_FMT_INT8: K * N + 2 * N, B200_FMT_INT4: K * N / 2 + K * N / group * 4}[fmt]
    nrot = max(2, int(300e6 // wbytes) + 1)
    ws_ = []
    for r in range(nrot):
        if fmt == B200_FMT_INT4:
            qp = torch.randint(0, 256, (K, N // 2), device=dev, dtype=torch.uint8)
            s = (torch.randn(K // group, N, device=dev).abs() * 0.01 + 1e-3).half()
            w = ops.pack_w4(qp, s, s, group, perm=torch.randperm(K) if act_order else None)
        elif fmt == B200_FMT_INT8:
            w = ops.pack_w8(torch.randint(-128, 128, (K, N), device=dev, dtype=torch.int8), torch.ones(N, device=dev).half())
        else:
            w = ops.PackedWeight(B200_FMT_F16, K, N, (torch.randn(N, K, device=dev) * 0.02).half())
        ws_.append(w)
    x = torch.randn(B, K, device=dev).half()
    y = torch.empty(B, N, device=dev).half()
    wk = ops.gemm_workspace(B, [(K, N)], dev)
    xp = torch.empty(B, K, device=dev).half() if act_order else None
    us = timeit(lambda i: ops.wo_gemm(x, ws_[i], wk, out=y, pdl=pdl, x_perm=xp), nrot)
    byt = wbytes + 2 * B * (K + N)
    for k in (env or {}):
        os.environ.pop(k, None)
    print(f"gemm {nm} B{B} K{K} N{N} {env or ''}{' pdl' if pdl else ''}{' act-order (gather + GEMM)' if act_order else ''}: {us:8.1f} us  {byt / us / 1e3:7.0f} GB/s  frac={byt / us / 1e3 / PEAK:.3f}",
          flush=True)
    return us


if __name__ == "__main__":
    which = sys.argv[1:] or ["attn", "gemm"]
    if which[0] == "one_gemm":     # one_gemm fmt B K N  (for ncu)
        f = {"f16": B200_FMT_F16, "int8": B200_FMT_INT8, "int4": B200_FMT_INT4}[which[1]]
        bench_gemm(f, int(which[2]), int(which[3]), int(which[4]))
        sys.exit(0)
    if which[0] == "one_attn":     # one_attn B Hq Hkv S
        bench_attn(int(which[1]), int(which[2]), int(which[3]), int(which[4]))
        sys.exit(0)
    import subprocess
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    print(torch.cuda.get_device_name(0), "power limit, max SM clock:", power or "unknown", "peak", PEAK)
    if "clusters" in which:
        # co-resident clusters of the INT4 g128 batch-pad-32 GEMM kernel: a split-K cluster of S CTAs needs S slots in ONE GPC
        import ctypes
        from rtp_llm_b200 import _lib
        for size in (1, 2, 4, 8):
            n = ctypes.c_int(0)
            _lib.check(_lib.load().b200_wo_gemm_max_active_clusters(size, ctypes.byref(n)), "wo_gemm_max_active_clusters")
            print(f"clusters of {size}: {n.value} co-resident ({n.value * size} CTAs, {torch.cuda.get_device_properties(0).multi_processor_count} SMs)",
                  flush=True)
    if "splits" in which:
        # o and w2 of Llama-3-8B at B32 with every split-K the plan may pick
        for K, N in ((4096, 4096), (14336, 4096)):
            for s in (1, 2, 4, 8):
                bench_gemm(B200_FMT_INT4, 32, K, N, env={"B200_GEMM_SPLITK": s})
    if "permute" in which:
        # GPTQ act-order: the x gather alone, then the Llama-3-8B INT4 GEMMs it precedes (qkv, o, w13) with and without it
        for K in (4096, 8192, 14336):
            bench_permute(32, K)
        for K, N in ((4096, 6144), (4096, 4096), (4096, 28672)):
            bench_gemm(B200_FMT_INT4, 32, K, N)
            bench_gemm(B200_FMT_INT4, 32, K, N, act_order=True)
    if "attn" in which:
        bench_attn(32, 32, 8, 2048)
        for c in (2, 4, 8, 16, 32):
            bench_attn(32, 32, 8, 2048, env={"B200_ATTN_TILES_PER_SPLIT": c})
        bench_attn(1, 32, 8, 4096)
        bench_attn(64, 32, 8, 4096)
        bench_attn(16, 8, 1, 8192)
    if "attn-multi" in which:
        # speculative-token verification at group 8 (Qwen2-72B / Llama-3-70B): 8, 16, 32, 64 query rows per kv head
        t = {n: bench_attn_multi(32, 64, 8, 2048, n) for n in (1, 2, 4, 8)}
        print("attn-multi time relative to q_len 2 (16 rows): " + ", ".join(f"q_len {n}: {t[n] / t[2]:.2f}x" for n in t), flush=True)
    if "attn-tree" in which or "tree-verify" in which or "kv-compact" in which:
        import subprocess
        print("tree benches on " + (subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                                                    "-i", "0"], capture_output=True, text=True).stdout.strip() or "unknown card")
              + " (name, power limit, SM clock, max SM clock)", flush=True)
    if "attn-tree" in which:
        # Llama-3-8B heads (group 4) at B 32, S 2048: the tree instance against the q_len instance on the same rows
        for n in (4, 8, 16):
            for kind in ("chain", "star", "binary"):
                bench_attn_tree(32, 32, 8, 2048, n, kind)
    if "tree-verify" in which:
        for B in (8, 32):
            for n in (4, 8, 16):
                for sampling in (False, True):
                    bench_tree_verify(B, n, sampling)
    if "kv-compact" in which:
        for B in (8, 32):
            bench_kv_compact(B)
    if "attn-beam" in which:
        # a request's beams in one CTA against one CTA per beam, Llama-3-8B heads (group 4) and group 8 at W 8
        import subprocess
        print("attn-beam on " + (subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                                                 "-i", "0"], capture_output=True, text=True).stdout.strip() or "unknown card")
              + " (name, power limit, SM clock, max SM clock)", flush=True)
        for B, W, Hq in ((8, 4, 32), (32, 4, 32), (4, 16, 32), (16, 8, 32), (16, 8, 64), (8, 2, 32), (8, 8, 32)):
            bench_attn_beam(B, W, Hq, 8)
    if "beam" in which:
        # beam search over Llama-3's vocabulary, with and without the 3-gram ban over 2048 history tokens, alternating
        for B, W in ((8, 4), (32, 4), (4, 16)):
            t = {n: [] for n in (0, 3)}
            for _ in range(3):
                for n in t:
                    t[n].append(bench_beam(B, W, ngram=n))
            print(f"beam B{B} W{W} V128256 median: step {sorted(t[0])[1]:.1f} us, ban n3 + step {sorted(t[3])[1]:.1f} us", flush=True)
    if "beam-hyps" in which:
        # the finished-hypothesis update and finalize at the beam step's shapes, short and long paths; medians of 3
        for B, W in ((8, 4), (32, 4), (4, 16)):
            for L in (16, 512):
                t = [bench_beam_hyps(B, W, L) for _ in range(3)]
                m = [sorted(x[k] for x in t)[1] for k in range(3)]
                print(f"beam-hyps B{B} W{W} max_len {L} median: update steady {m[0]:.2f} us, empty (+ memset) {m[1]:.2f} us, "
                      f"finalize {m[2]:.2f} us", flush=True)
    if "logprobs" in which:
        # the log-prob kernel over Llama-3's vocabulary at B 32: the drawn token's log-prob alone, and with the top 5 / 20
        t = {n: sorted(bench_logprobs(32, n) for _ in range(3))[1] for n in (0, 5, 20)}
        print("logprobs B32 V128256 median: " + ", ".join(f"top_n {n}: {v:.1f} us" for n, v in t.items()), flush=True)
    if "sample" in which:
        # b200_sample alone (one 1024-thread CTA per row, bisection passes over the vocabulary): top-k 50 and top-p 0.9 each
        # and together, minus the logit copy the in-place op needs before every call
        for B in (8, 32):
            c = sorted(bench_sample(B, 0, 1.0, copy_only=True) for _ in range(3))[1]
            for k, p in ((50, 1.0), (0, 0.9), (50, 0.9)):
                m = sorted(bench_sample(B, k, p) for _ in range(3))[1]
                print(f"sample B{B} V128256 top_k {k} top_p {p} median: {m - c:.1f} us (copy + sample {m:.1f}, copy {c:.1f})",
                      flush=True)
    if "sample-min-p" in which:
        # b200_sample with and without a min_p buffer (top-p 0.9, min_p 0.05), alternating, minus the logit copy; medians of 3
        for B in (8, 32):
            c = sorted(bench_sample(B, 0, 1.0, copy_only=True) for _ in range(3))[1]
            t = {m: [] for m in (None, 0.05)}
            for _ in range(3):
                for m in t:
                    t[m].append(bench_sample(B, 0, 0.9, min_p=m))
            off, on = sorted(t[None])[1] - c, sorted(t[0.05])[1] - c
            print(f"sample B{B} V128256 top_p 0.9 median: min_p off {off:.1f} us, min_p 0.05 {on:.1f} us ({on - off:+.1f} us)",
                  flush=True)
    if "constrain" in which:
        # the grammar mask and logit bias over Llama-3's and Qwen's vocabularies at B 32 / 128, fp16 logits; medians of 3
        for V in (128256, 151936):
            for rows in (32, 128):
                for mask in ("ones", "half", "single"):
                    for bias in (0, 300):
                        m = sorted(bench_constrain(rows, V, mask, bias) for _ in range(3))[1]
                        print(f"constrain rows {rows} V{V} mask {mask} bias {bias}/row median: {m:.2f} us", flush=True)
    if "rope" in which:
        # Llama-3 shape (Hq 32, Hkv 8, D 128) at B 32: the Base-only kernel against the full-contract kernel, 1 and 4 tokens
        for n in (1, 4):
            t = {k: bench_rope(k, 32, 32, 8, n) for k in ("base", "llama3", "yarn table")}
            print(f"rope q_len {n} relative to base: " + ", ".join(f"{k}: {t[k] / t['base']:.2f}x" for k in t), flush=True)
    if "qknorm-rope" in which:
        # Qwen3-8B's attention shape (Hq 32, Hkv 8, D 128) at B 32: the fused QK-norm + rope against the two launches, alternating
        for kind in ("base", "yarn table"):
            for n in (1, 4):
                t = {f: [] for f in (True, False)}
                for _ in range(3):
                    for f in t:
                        t[f].append(bench_qknorm_rope(kind, f, 32, 32, 8, n))
                fu, co = sorted(t[True])[1], sorted(t[False])[1]
                print(f"qknorm-rope {kind} q_len {n} median: fused {fu:.2f} us, norm + rope {co:.2f} us ({fu / co:.2f}x)", flush=True)
    if "gemm" in which:
        for B in (32,):
            bench_gemm(B200_FMT_INT4, B, 4096, 6144)
            bench_gemm(B200_FMT_INT4, B, 4096, 4096)
            bench_gemm(B200_FMT_INT4, B, 4096, 28672)
            bench_gemm(B200_FMT_INT4, B, 14336, 4096)
        bench_gemm(B200_FMT_INT4, 32, 4096, 28672, pdl=True)
        bench_gemm(B200_FMT_INT4, 1, 4096, 28672)
        bench_gemm(B200_FMT_INT4, 64, 4096, 28672)
        for group in (64, 32):                        # GPTQ / AWQ checkpoints with finer groups, same Llama-3-8B shapes
            bench_gemm(B200_FMT_INT4, 32, 4096, 6144, group=group)
            bench_gemm(B200_FMT_INT4, 32, 4096, 4096, group=group)
            bench_gemm(B200_FMT_INT4, 32, 4096, 28672, group=group)
            bench_gemm(B200_FMT_INT4, 32, 14336, 4096, group=group)
            bench_gemm(B200_FMT_INT4, 1, 4096, 28672, group=group)
            bench_gemm(B200_FMT_INT4, 64, 4096, 28672, group=group)
        bench_gemm(B200_FMT_INT8, 32, 4096, 28672)
        bench_gemm(B200_FMT_F16, 32, 4096, 28672)
        bench_gemm(B200_FMT_F16, 32, 4096, 128256)
