"""GPU tests (H100) of beam search: b200_beam_search_step and b200_ban_repeat_ngram against the float64 reference
(tests/beam_oracle.py), their bits under CUDA-graph replay with PDL, and DecodeStep's beam mode: the step's logits and
selections, the page-table fork (bit-exact K/V histories), a re-score of the surviving beams through plain steps, and
beam_width 1 against the greedy step."""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200.decode_step import TINY, DecodeStep  # noqa: E402
from tests.beam_oracle import banned_np, beam_step_np, check_beam, score_tol  # noqa: E402
from tests.step_oracle import bits, check_logits, device_state, oracle_step  # noqa: E402

DEV = torch.device("cuda")
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _case(B, W, V, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * W, V, generator=g) * 3.0
    x[0, ::7] = -float("inf")                                    # masked logits
    if W > 1:
        x[1] = x[0]                                              # exact duplicates across beams (equal cum below)
    if B > 1:
        x[W, : V - 2 * W + 1] = -float("inf")                   # fewer than 2W finite logits in one row
    x = x.to(dtype)
    cum = -torch.rand(B, W, generator=g) * 4.0
    if W > 1:
        cum[0, 1] = cum[0, 0]
    if B > 1:
        cum[1, 1:] = -float("inf")                               # first step of request 1
    return x, cum


@pytest.mark.parametrize("V", [64, 1000, 32000, 128256, 152064])
@pytest.mark.parametrize("W", [1, 2, 4, 8, 16, 32])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_beam_step_vs_float64_reference(dt, W, V):
    B = 3
    x, cum = _case(B, W, V, DTYPES[dt], seed=W * 7 + V)
    x64 = x.double().numpy()
    eos = int(beam_step_np(x64, cum.numpy())["cand_token"][0, 0])   # request 0's best candidate is EOS
    exp = beam_step_np(x64, cum.numpy(), eos_id=eos)
    out = ops.beam_search_step(x.to(DEV), cum.to(DEV), W, eos_id=eos)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    check_beam(got, exp, W, eos)
    assert got["cand_token"][0, 0] == eos and eos not in got["next_token"][0]


def test_width_one_picks_the_argmax_token():
    B, V = 64, 128256
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(B, V, generator=g) * 2.0).to(torch.float16)
    cum = -torch.rand(B, 1, generator=g)
    out = ops.beam_search_step(x.to(DEV), cum.to(DEV), 1)
    am = ops.argmax(x.to(DEV)).cpu().numpy()
    torch.cuda.synchronize()
    exp = beam_step_np(x.double().numpy(), cum.numpy())
    rs = exp["ranked_scores"]
    clear = rs[:, 0].astype(np.float32) != rs[:, 1].astype(np.float32)
    assert clear.sum() > B // 2
    nt = out["next_token"].cpu().numpy()[:, 0]
    np.testing.assert_array_equal(nt[clear], am[clear])
    nc = out["next_cum"].cpu().numpy()[:, 0].astype(np.float64)
    x64 = x.double().numpy()
    ls = x64[np.arange(B), am] - (x64.max(1) + np.log(np.exp(x64 - x64.max(1, keepdims=True)).sum(1)))
    e = cum.numpy()[:, 0] + ls
    assert (np.abs(nc - e)[clear] <= score_tol(e)[clear]).all()


@pytest.mark.parametrize("dt", list(DTYPES))
def test_ngram_ban_is_exact(dt):
    rows, V, stride = 24, 1000, 8192
    rng = np.random.default_rng(5)
    hist = rng.integers(0, 12, (rows, stride)).astype(np.int32)          # a small alphabet: many repeated n-grams
    hist[rng.random((rows, stride)) < 0.02] = -5                          # out-of-range ids
    hist[rng.random((rows, stride)) < 0.02] = V + 3
    hist[:, :64] += rng.integers(0, 900, (rows, 1)).astype(np.int32)    # some distinct ids per row
    L = np.array([0, 1, 2, 7, 8, 9, 100, 4096, 8191, 8192, 8192, 5000] * 2, np.int32)
    n = np.array([1, 2, 3, 4, 5, 6, 7, 8, 1, 2, 3, 8, 0, -1, 2, 3, 4, 5, 6, 7, 8, 1, 2, 3], np.int32)
    x = (torch.randn(rows, V, generator=torch.Generator().manual_seed(6)) * 3).to(DTYPES[dt])
    got = ops.ban_repeat_ngram(x.to(DEV), torch.from_numpy(hist).to(DEV), torch.from_numpy(L).to(DEV),
                               torch.from_numpy(n).to(DEV)).cpu()
    exp = banned_np(hist, L, n, V)
    assert sum(e.size for e in exp) > 50
    for r in range(rows):
        ninf = np.nonzero(torch.isneginf(got[r]).numpy())[0]
        np.testing.assert_array_equal(ninf, exp[r], err_msg=f"row {r} (n {n[r]}, L {L[r]})")
        keep = np.ones(V, bool)
        keep[exp[r]] = False
        k = torch.from_numpy(keep)
        assert torch.equal(_bits(got[r][k]), _bits(x[r][k])), f"row {r}: other logits changed"


def test_both_ops_give_the_same_bits_under_graph_replay_with_pdl():
    B, W, V, stride = 8, 4, 128256, 2048
    x, cum = _case(B, W, V, torch.float16, seed=3)
    src, cum = x.to(DEV), cum.to(DEV)
    rng = np.random.default_rng(8)
    hist = torch.from_numpy(rng.integers(0, 50, (B * W, stride)).astype(np.int32)).to(DEV)
    hl = torch.full((B * W,), stride, dtype=torch.int32, device=DEV)
    ng = torch.full((B * W,), 3, dtype=torch.int32, device=DEV)
    logits = torch.empty_like(src)
    ws = ops.beam_search_workspace(B, W, V, DEV)
    outs = {k: torch.empty((B, n), dtype=d, device=DEV) for k, n, d in (
        ("cand_token", 2 * W, torch.int32), ("cand_parent", 2 * W, torch.int32), ("cand_score", 2 * W, torch.float32),
        ("next_token", W, torch.int32), ("next_parent", W, torch.int32), ("next_cum", W, torch.float32))}

    def run():
        logits.copy_(src)
        ops.ban_repeat_ngram(logits, hist, hl, ng)
        ops.beam_search_step(logits, cum, W, eos_id=5, workspace=ws, out=outs)

    def snap():
        torch.cuda.synchronize()
        return [logits.clone()] + [v.clone() for v in outs.values()]
    run()
    ref = snap()
    run()
    assert all(torch.equal(a, b) for a, b in zip(ref, snap())), "repeated eager calls differ"
    ops.set_pdl(True)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            run()
        for _ in range(3):
            for v in outs.values():
                v.fill_(-7)
            graph.replay()
            assert all(torch.equal(a, b) for a, b in zip(ref, snap())), "graph replay with PDL differs"
    finally:
        ops.set_pdl(False)
    assert int(ws[:4 * (B * W + B)].view(torch.int32).abs().sum()) == 0, "arrival counters not reset"


# ---------------------------------------------------------------------------------------------------- decode step
def _seed_history(model, n):
    """A prompt history whose last n - 1 ids (ending in each row's input token) occurred once before, followed by a row-specific
    token: with the n-gram ban on, step 1 must ban that token in every row (n == 1 bans the input token itself)."""
    ids = model.ids.cpu().tolist()
    rows = []
    for r, a in enumerate(ids):
        if n <= 1:
            rows.append([a])
            continue
        pre = [7] * (n - 2) + [a]
        rows.append(pre + [(a + 1 + r) % model.vocab] + pre)
    L = len(rows[0])
    model.hist[:, :L] = torch.tensor(rows, dtype=torch.int32, device=DEV)
    model.hist_len.fill_(L)
    return rows


STEP = [("int4", "eager", 0), ("f16", "eager", 1), ("int4", "graph pdl", 2), ("f16", "graph pdl", 3)]


@pytest.mark.parametrize("case", STEP, ids=[f"{q} {m} ngram {n}" for q, m, n in STEP])
def test_beam_step_vs_oracle(case):
    """Each step: the logits against oracle_step on the state the step started from, with the n-gram ban the reference
    predicts from the step's history applied to the ORACLE's logits -- the step's -inf positions must be exactly those, every
    other logit within the step tolerance; the selection against the reference on the step's logits; and after the fork,
    every row's token history equal to its beam's token path (the seeded prompt history, then the next_parent chain)."""
    quant, mode, ngram = case
    cfg = dataclasses.replace(TINY, quant=quant)
    W, steps = 4, 6
    model = DecodeStep(cfg, 2, 40, DEV, keep_reference=True, ragged=True, seed=4, pdl="pdl" in mode, beam_width=W,
                       no_repeat_ngram=ngram)
    R, V = model.B, model.vocab
    try:
        if "graph" in mode:
            model.capture()
        model.upload_inputs()
        paths = _seed_history(model, ngram)
        bans = []
        for t in range(steps):
            torch.cuda.synchronize()
            state, kv_before = device_state(model), [bits(L["kv"]) for L in model.layers]
            cum = model.beam_cum.cpu().numpy()
            hist, hist_len = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
            model.replay() if "graph" in mode else model.run()
            torch.cuda.synchronize()
            got = model.logits.float().cpu().numpy()
            exp = oracle_step(state, kv_before)
            banned = banned_np(hist, hist_len, [ngram] * R, V) if ngram > 0 else [np.zeros(0, np.int64)] * R
            bans.append(sum(b.size for b in banned))
            fin = np.ones_like(got, dtype=bool)
            for r in range(R):
                np.testing.assert_array_equal(np.nonzero(np.isneginf(got[r]))[0], banned[r], err_msg=f"step {t} row {r}: banned set")
                fin[r, banned[r]] = False
            check_logits(got, exp, mask=fin)
            sel = {k: v.cpu().numpy() for k, v in model.beam_out.items()}
            check_beam(sel, beam_step_np(got, cum), W, -1)
            par = (np.arange(R) // W * W + sel["next_parent"].reshape(-1)).tolist()
            paths = [paths[par[j]] + [int(sel["next_token"].reshape(-1)[j])] for j in range(R)]
            h, hl = model.hist.cpu().numpy(), model.hist_len.cpu().numpy()
            for j in range(R):
                assert hl[j] == len(paths[j]) and h[j, :hl[j]].tolist() == paths[j], f"step {t} row {j}: token history"
        if ngram > 0:
            assert bans[0] >= R, bans                  # the seeded history bans at least one token per row at step 1
    finally:
        ops.set_pdl(False)


def test_fork_gives_every_beam_its_ancestry_bit_for_bit():
    """8 steps of W 4 with page crossings (tokens_per_block 16). Before each fork the K/V slot each row just wrote is
    recorded; after it, every beam's visible slots 0..seq through its page table must be the prompt's slots followed by
    the recorded slots of its ancestry (the next_parent chain)."""
    W, steps, T = 4, 8, TINY.tokens_per_block
    model = DecodeStep(dataclasses.replace(TINY, quant="int4"), 2, 40, DEV, ragged=True, seed=6, beam_width=W)
    R = model.B
    seq0 = model.seq_lens.cpu().long()
    assert ((seq0 + steps) // T > seq0 // T).any(), "no page crossing in this run"
    prompt_tbl = model.block_ids.clone()

    def slots(kv, tbl, n):                                       # [n, 2, Hkv, D] of slots 0..n-1 through the table row tbl
        x = torch.arange(n, device=DEV)
        return kv[tbl[x // T].long(), :, :, x % T, :]
    prompt = [[slots(L["kv"], prompt_tbl[r], int(seq0[r])).clone() for L in model.layers] for r in range(R)]
    chain = [[[] for _ in model.layers] for _ in range(R)]
    written, moved = {}, False
    fork = model.fork

    def recording_fork():
        seq, tbl = model.seq_lens.clone().long(), model.block_ids.clone()
        for li, L in enumerate(model.layers):
            written[li] = [L["kv"][tbl[r, seq[r] // T].long(), :, :, seq[r] % T, :].clone() for r in range(R)]
        fork()
    model.fork = recording_fork
    for _ in range(steps):
        model.run()
        torch.cuda.synchronize()
        parent = (torch.arange(R) // W * W + model.beam_out["next_parent"].cpu().view(-1)).tolist()
        moved |= any(parent[j] != j for j in range(R))
        chain = [[chain[parent[j]][li] + [written[li][parent[j]]] for li in range(len(model.layers))] for j in range(R)]
        seq, tbl = model.seq_lens.cpu().long(), model.block_ids
        for j in range(R):
            assert int(seq[j]) == int(seq0[j]) + len(chain[j][0])
            for li, L in enumerate(model.layers):
                exp = torch.cat([prompt[j][li]] + [c.unsqueeze(0) for c in chain[j][li]])
                assert torch.equal(slots(L["kv"], tbl[j], int(seq[j])), exp), f"beam {j} layer {li}: K/V history differs"
    assert moved, "no beam ever changed parent: the fork was not exercised"


def test_surviving_beams_rescore_through_plain_steps():
    """Each surviving beam's tokens fed through plain (greedy) steps as forced inputs, with a cache of their own that starts
    as a copy of the prompt pages: the float64 log-softmax of each next token, summed, must match the beam's cum_log_probs.
    Both runs push the same token paths through the same kernels at the same row count; a path's tokens may sit in other
    rows of the GEMM tiles than in the beam run (its ancestors moved between rows), which changes nothing in a row's sum.
    What is left is fp32 against float64 in the log-softmax and the fp16 logits' rounding: far below the 1e-2 per step
    allowed here."""
    W, steps = 4, 6
    cfg = dataclasses.replace(TINY, quant="int4")
    beam = DecodeStep(cfg, 2, 40, DEV, ragged=True, seed=7, beam_width=W)
    plain = DecodeStep(cfg, 2 * W, 40, DEV, ragged=True, seed=7)
    R = beam.B
    plain.block_ids_h.copy_(beam.block_ids_h)
    plain.seq_lens_h.copy_(beam.seq_lens_h)
    for Lp, Lb in zip(plain.layers, beam.layers):
        Lp["kv"].copy_(Lb["kv"])
    paths = [[int(t)] for t in beam.ids_h.tolist()]
    for _ in range(steps):
        beam.run()
        torch.cuda.synchronize()
        par = (torch.arange(R) // W * W + beam.beam_out["next_parent"].cpu().view(-1)).tolist()
        tok = beam.beam_out["next_token"].cpu().view(-1).tolist()
        paths = [paths[par[j]] + [tok[j]] for j in range(R)]
    cum = beam.beam_cum.cpu().numpy().reshape(-1).astype(np.float64)
    score = np.zeros(R)
    for t in range(steps):
        plain.ids_h.copy_(torch.tensor([p[t] for p in paths], dtype=torch.int32))
        plain.seq_lens_h.copy_(beam.seq_lens_h + t)
        plain.upload_inputs()
        plain.run()
        torch.cuda.synchronize()
        x = plain.logits.double().cpu().numpy()
        m = x.max(1, keepdims=True)
        ls = x - m - np.log(np.exp(x - m).sum(1, keepdims=True))
        score += ls[np.arange(R), [p[t + 1] for p in paths]]
    assert np.abs(score - cum).max() <= 1e-2 * steps, (score, cum)


def test_width_one_is_the_greedy_step():
    cfg = dataclasses.replace(TINY, quant="int4")
    a = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=9)
    b = DecodeStep(cfg, 4, 40, DEV, ragged=True, seed=9, beam_width=1)
    for _ in range(3):
        for m in (a, b):
            m.run()
        torch.cuda.synchronize()
        assert torch.equal(a.next_ids, b.next_ids) and torch.equal(a.logits, b.logits)
        # the beam kernel at W 1 on the step's logits picks the greedy token wherever the top two are apart in fp32
        out = ops.beam_search_step(a.logits, torch.zeros(4, 1, device=DEV), 1)
        x = a.logits.double().cpu().numpy()
        srt = np.sort(x, 1)
        clear = srt[:, -1].astype(np.float32) != srt[:, -2].astype(np.float32)
        np.testing.assert_array_equal(out["next_token"].cpu().numpy()[clear, 0], a.next_ids.cpu().numpy()[clear])
        for m in (a, b):
            m.ids_h.copy_(a.next_ids.cpu())
            m.seq_lens_h += 1
            m.upload_inputs()


def test_beam_step_is_not_a_program():
    model = DecodeStep(TINY, 2, 40, DEV, beam_width=2)
    with pytest.raises(ValueError, match="program"):
        model.build_program()
