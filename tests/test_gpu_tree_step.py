"""GPU tests (H100) of DecodeStep's token-tree mode: a chain tree is the chain verification step bit for bit; a tree whose greedy
branch is not the first child accepts the plain steps' tokens along that branch; the verifier's decisions are those of
tests/verify_oracle.py on the step's own rows; and after the step the accepted path's K/V sit at slots seq .. seq + accepted."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep, SamplingParams  # noqa: E402
from tests.step_oracle import TINY31, check_logits  # noqa: E402
from tests.verify_oracle import verify_np  # noqa: E402

DEV = torch.device("cuda")
MODES = ["eager", "graph", "pdl", "graph pdl"]


def _run(model, mode):
    try:
        if "graph" in mode:
            model.capture()
            model.replay()
        else:
            model.run()
        torch.cuda.synchronize()
    finally:
        ops.set_pdl(False)


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
@pytest.mark.parametrize("mode", MODES)
def test_chain_tree_step_is_the_chain_step_bit_for_bit(mode, sampled):
    samp = SamplingParams(temperature=0.8, top_k=50, top_p=0.9, seed=3) if sampled else None
    kw = dict(ragged=True, seed=2, q_len=4, pdl="pdl" in mode, sampling=samp)
    outs = []
    for tree in (None, [-1, 0, 1, 2]):
        m = DecodeStep(TINY31, 4, 40, DEV, tree=tree, **kw)
        _run(m, mode)
        outs.append((m.logits.clone(), m.out_tokens.clone(), m.accepted.clone(), [L["kv"].clone() for L in m.layers],
                     getattr(m, "accepted_path", None)))
    (l0, o0, a0, kv0, _), (l1, o1, a1, kv1, p1) = outs
    assert torch.equal(l0.view(torch.int16), l1.view(torch.int16)), "logits differ"
    assert torch.equal(o0, o1) and torch.equal(a0, a1), (o0, o1, a0, a1)
    assert all(torch.equal(x.view(torch.int16), y.view(torch.int16)) for x, y in zip(kv0, kv1)), "caches differ"
    a = a1.cpu().numpy()
    np.testing.assert_array_equal(p1.cpu().numpy(), [[i if i <= a[b] else -1 for i in range(4)] for b in range(4)])


# node 0 the root; node 1 a decoy under it, node 2 plain step 1's input; node 3 a decoy under node 2, node 4 plain step 2's input
BRANCH = [-1, 0, 0, 2, 2]


@pytest.mark.parametrize("mode", MODES[:3])
@pytest.mark.parametrize("cfg", [dataclasses.replace(TINY, quant="int4"), dataclasses.replace(TINY, quant="f16"), TINY31],
                         ids=["int4", "f16", "llama31"])
def test_tree_step_follows_the_greedy_branch_of_plain_steps(cfg, mode):
    """Two greedy single-token steps on one model, then one tree step on an identical model whose second child of the root and
    second child of that node carry those tokens and whose first children are decoys. The path rows' logits match the plain
    steps; where every plain step's top-2 margin is clear of the error, the tree accepts 2 along [0, 2, 4] and emits plain step
    2's token; everywhere the decisions are verify_np's on the step's own rows; and the K/V of nodes 2 and 4 end at slots
    seq + 1 and seq + 2."""
    plain = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2)
    tree = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2, q_len=5, tree=BRANCH, pdl="pdl" in mode)
    plain.seq_lens_h.copy_(tree.seq_lens_h)
    plain.ids_h.copy_(tree.ids_h[:, 0])
    toks, logits = [plain.ids_h.clone()], []
    for _ in range(3):
        plain.upload_inputs()
        plain.run()
        torch.cuda.synchronize()
        logits.append(plain.logits.float().cpu().numpy())
        toks.append(plain.next_ids.cpu())
        plain.ids_h.copy_(plain.next_ids.cpu())
        plain.seq_lens_h += 1
    V = cfg.vocab
    tree.ids_h.copy_(torch.stack([toks[0], (toks[1] + 1) % V, toks[1], (toks[2] + 1) % V, toks[2]], dim=1))
    tree.upload_inputs()
    _run(tree, mode)
    got = tree.logits.float().cpu().numpy().reshape(tree.B, 5, -1)[:, [0, 2, 4]]
    exp = np.stack(logits, axis=1)
    err = check_logits(got, exp)
    srt = np.sort(exp, axis=-1)
    sure = ((srt[..., -1] - srt[..., -2]) > 2 * err + 1e-6).all(axis=1)
    assert sure.any(), "no sequence with a clear margin at every step"
    acc, out, path = tree.accepted.cpu().numpy(), tree.out_tokens.cpu().numpy(), tree.accepted_path.cpu().numpy()
    assert (acc[sure] == 2).all(), acc
    assert (path[sure] == [0, 2, 4, -1, -1]).all(), path
    np.testing.assert_array_equal(out[sure, :3], torch.stack(toks[1:4], dim=1).numpy()[sure])
    eo, ea, ep, _ = verify_np(np.tile(BRANCH, (tree.B, 1)), tree.ids_h.numpy(), target_ids=tree.next_ids.view(tree.B, 5).cpu().numpy())
    np.testing.assert_array_equal(acc, ea)
    np.testing.assert_array_equal(out, eo)
    np.testing.assert_array_equal(path, ep)
    # the compaction: against the same step run without it, slot seq + d holds node path[d]'s K/V and nothing else changed
    raw = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=2, q_len=5, tree=BRANCH)
    raw.ids_h.copy_(tree.ids_h)
    raw.upload_inputs()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "kv_compact_path", lambda *a, **k: None)
        _run(raw, "eager")
    seq, T, bl = tree.seq_lens_h.numpy(), cfg.tokens_per_block, tree.block_ids_h.numpy()
    for L, R in zip(tree.layers, raw.layers):
        exp = R["kv"].view(torch.int16).cpu().numpy()
        src = exp.copy()
        for b in range(tree.B):
            slot = lambda q: (bl[b, q // T], slice(None), slice(None), q % T)
            for d in range(1, acc[b] + 1):
                exp[slot(int(seq[b]) + d)] = src[slot(int(seq[b]) + path[b, d])]
        np.testing.assert_array_equal(L["kv"].view(torch.int16).cpu().numpy(), exp)
