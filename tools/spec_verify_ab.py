#!/usr/bin/env python
"""Bit identity of the speculative verifiers between two builds of the library (developer tool, runs on the GPU).

    python tools/spec_verify_ab.py LIB_A LIB_B

runs every verification entry (b200_spec_verify, b200_spec_verify_tree, b200_spec_verify_tree_draft) and every accept rule
(greedy, deterministic drafts, draft rows) on the same seeded inputs under each library, one process per library through
B200_LIB_PATH, and compares out_tokens, accepted and accepted_path bit for bit. The inputs: chains of 2 to 17 nodes, random,
binary and star trees up to 64 nodes, V 128256, 4096 and 1001, and target and draft rows 4 bytes off 16-byte alignment.
Exit status 1 when any output differs."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
dev = torch.device("cuda:0")


def _parents(rng, kind, n):
    return np.array([-1] + [{"chain": c - 1, "star": 0, "binary": (c - 1) // 2, "random": int(rng.integers(0, c))}[kind]
                            for c in range(1, n)], np.int32)


def _rows(g, shape, V):
    """Temperature-0.25 softmaxes, every third row sparse (its 40 largest entries), as fp32 on the device."""
    t = torch.softmax(torch.randn(*shape, V, generator=g) * 4, -1)
    flat = t.view(-1, V)
    sparse = flat[::3]
    keep = sparse.topk(min(40, V), -1).indices
    flat[::3] = torch.zeros_like(sparse).scatter_(-1, keep, sparse.gather(-1, keep))
    return (t / t.sum(-1, keepdim=True)).to(dev)


def _misalign(x):
    """x in a buffer 4 bytes past a 16-byte boundary."""
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device=dev)
    out = flat[1:].view(x.shape)
    out.copy_(x)
    return out


def _case(seed, kind, n, B, V, misaligned):
    """Target rows, draft rows (half the parent's target row, half another softmax; row 0 unread), node tokens (the argmax of
    the parent's target row for every third node, else drawn from the node's draft row; duplicate siblings under one root;
    one token outside the vocabulary) and uniforms."""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    par = np.stack([_parents(rng, kind, n) for _ in range(B)])
    t = _rows(g, (B, n), V)
    pidx = torch.from_numpy(par.clip(min=0)).long().to(dev)
    parent_rows = t.gather(1, pidx[..., None].expand(B, n, V))
    d = (0.5 * parent_rows + 0.5 * _rows(g, (B, n), V)).contiguous()
    d[:, 0] = float("nan")
    drawn = torch.multinomial(d[:, 1:].reshape(-1, V).nan_to_num(), 1, generator=torch.Generator(dev).manual_seed(seed))
    toks = torch.full((B, n), -1, dtype=torch.int32, device=dev)
    toks[:, 1:] = drawn.view(B, n - 1).to(torch.int32)
    best = parent_rows.argmax(-1).to(torch.int32)
    third = (torch.arange(n, device=dev) % 3 == 1)
    third[0] = False
    toks[:, third] = best[:, third]
    kids0 = [c for c in range(1, n) if par[0, c] == 0]
    for c in kids0[1:]:
        toks[0, c] = toks[0, kids0[0]]
    if B > 1:
        toks[1, n - 1] = V + 5
    u = torch.rand(B, n, generator=g).to(dev)
    ids = t.argmax(-1).to(torch.int32)
    if misaligned:
        t, d = _misalign(t), _misalign(d)
    return torch.from_numpy(par).to(dev), toks, t, d, u, ids


def cases():
    out = []
    for V in (4096, 1001):
        out += [("chain", n, 8, V, False) for n in range(2, 18)]
        out += [(k, n, 8, V, False) for k in ("random", "binary", "star") for n in (2, 5, 16, 33, 64)]
    out += [("chain", n, 8, 128256, False) for n in (2, 4, 8, 17)]
    out += [(k, n, 8, 128256, False) for k in ("random", "binary", "star") for n in (8, 64)]
    out += [("chain", 8, 8, 4096, True), ("random", 16, 8, 4096, True), ("binary", 31, 8, 4096, True)]
    return out


def dump(path):
    from rtp_llm_b200 import ops
    res = {}
    for i, (kind, n, B, V, mis) in enumerate(cases()):
        par, toks, t, d, u, ids = _case(1000 + i, kind, n, B, V, mis)
        name = f"{kind} n{n} B{B} V{V}{' misaligned' if mis else ''}"
        runs = {"tree greedy": lambda: ops.spec_verify_tree(par, toks, target_ids=ids),
                "tree deterministic": lambda: ops.spec_verify_tree(par, toks, target_probs=t, uniform=u),
                "tree draft rows": lambda: ops.spec_verify_tree(par, toks, target_probs=t, uniform=u, draft_probs=d)}
        if kind == "chain":
            dt, dp = toks[:, 1:].contiguous(), d[:, 1:].contiguous()
            runs["chain greedy"] = lambda: ops.spec_verify(dt, target_ids=ids)
            runs["chain deterministic"] = lambda: ops.spec_verify(dt, target_probs=t, uniform=u)
            runs["chain draft rows"] = lambda: ops.spec_verify(dt, target_probs=t, uniform=u, draft_probs=dp)
        for rule, fn in runs.items():
            for k, x in zip(("out_tokens", "accepted", "accepted_path"), fn()):
                res[f"{name} | {rule} | {k}"] = x.cpu().numpy()
    torch.cuda.synchronize()
    np.savez(path, **res)


def main():
    if sys.argv[1] == "--dump":
        dump(sys.argv[2])
        return 0
    libs = sys.argv[1:3]
    with tempfile.TemporaryDirectory() as tmp:
        got = []
        for j, lib in enumerate(libs):
            path = os.path.join(tmp, f"{j}.npz")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", path],
                                  env=dict(os.environ, B200_LIB_PATH=os.path.abspath(lib)))
            got.append(dict(np.load(path)))
    a, b = got
    assert a.keys() == b.keys()
    bad = [k for k in a if not np.array_equal(a[k], b[k])]
    runs = sorted({k.rsplit(" | ", 1)[0] for k in a})
    rules = sorted({k.split(" | ")[1] for k in a})
    for rule in rules:       # the decisions are not all alike: some walks accept, some stop at the root
        acc = np.concatenate([a[f"{r} | accepted"] for r in runs if r.split(" | ")[1] == rule])
        print(f"{rule}: {acc.size} sequences, accepted mean {acc.mean():.2f}, none accepted {(acc == 0).mean():.2f}")
    print(f"{len(runs)} runs ({len(a)} arrays): {len(a) - len(bad)} equal, {len(bad)} differ")
    for k in bad[:20]:
        print("DIFFERS:", k)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
