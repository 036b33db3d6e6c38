#!/usr/bin/env python
"""TP parity on real GPUs (developer tool; launch with torchrun --nproc-per-node N): the tiny decode step with the
reference's TP split over N ranks (NCCL all-reduce / all-gather) must match the UNSHARDED CPU oracle."""
import dataclasses
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rtp_llm_b200.decode_step import TINY, DecodeStep  # noqa: E402
from rtp_llm_b200.tp import make_comm  # noqa: E402
from tests import step_oracle  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=dev)
    comm = make_comm(dev, kind=os.environ.get("B200_COMM", "peer"))
    ok = True
    for quant in ("int4", "int8", "f16"):
        cfg = dataclasses.replace(TINY, quant=quant, head_num=8, kv_head_num=2 if world <= 2 else world, hidden=1024,
                                  inter=1024, vocab=1000)
        model = DecodeStep(cfg, 5, 70, dev, tp_rank=rank, tp_size=world, comm=comm, keep_reference=True, ragged=True, seed=2)
        # the oracle runs unsharded: TP=1 twin with the same seeds (weights are generated full, then sliced per rank)
        kv_before = None
        if os.environ.get("TP_PROGRAM", "0") == "1" and hasattr(comm, "argmax"):
            model.build_program()
        model.capture()
        for _ in range(3):
            model.replay()
        torch.cuda.synchronize()
        dist.all_gather_into_tensor(model.logits_all, model.logits)
        logits = model.logits_all.permute(1, 0, 2).reshape(model.B, -1)[:, : cfg.vocab].float().cpu().numpy()
        tok = model.next_ids.cpu().numpy()
        toks = [None] * world
        dist.all_gather_object(toks, tok.tolist())
        if rank == 0:
            # assemble the unsharded model view for the oracle
            full = types_ns(model, cfg, kv_before, world)
            exp = step_oracle.oracle_step(full, full.kv_before)
            err, bound = step_oracle.logit_error(logits, exp)
            good = err <= bound
            # sampled tokens: identical on every rank, equal to the argmax of the gathered logits
            good &= all(t == toks[0] for t in toks) and toks[0] == np.argmax(logits, axis=-1).tolist()
            ok &= good
            print(f"[{'PASS' if good else 'FAIL'}] tp{world} {quant}: max logit err {err:.4g} (bound {bound:.3g})", flush=True)
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    os._exit(0 if ok else 1)


def types_ns(model, cfg, kv_before, world):
    """An object with the attributes oracle_step() reads, describing the UNSHARDED model (full weights, full KV pool: every
    rank generated the full pool from a common seed and kept only ITS kv heads, so ranks hold different K/V)."""
    import types
    full = types.SimpleNamespace()
    full.cfg, full.B, full.D, full.q_len, full.rope_spec = cfg, model.B, model.D, model.q_len, model.rope_spec
    full.Hq, full.Hkv = cfg.head_num, cfg.kv_head_num
    full.ids_h, full.seq_lens_h, full.block_ids_h = model.ids_h, model.seq_lens_h, model.block_ids_h
    full.embed, full.final_ln = model.embed, model.final_ln
    full.lm_head_ref = model.lm_head_full
    full.layers = [dict(ln1=L["ln1"], ln2=L["ln2"], ref=L["full"]) for L in model.layers]
    full.kv_before = [step_oracle.bits(L["kv_full"]) for L in model.layers]
    return full


if __name__ == "__main__":
    main()
