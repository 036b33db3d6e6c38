"""GPU tests (H100) of what happens between the ops of one persistent-kernel launch (csrc/decode_program.cuh): grid barriers,
the arrival wait, the proxy fence at each op end, rings whose counters run on across ops, split-K state shared by
consecutive GEMMs, and the segment breaks of the recorder.

Each chain of tests/program_chains.py is recorded twice: as it is, and with a separator (one argmax launch on a private
scratch row) after every persistent-capable call, so that in the reference every persistent op is a segment of its own and
runs through the same b200_program_launch path. An op's plan does not depend on its neighbours, so the two programs must give
the same bits in every output and every in-place buffer; the one-op form is pinned to float64 by test_gpu_gemm_exact.py and
test_gpu_glue_exact.py. Before each launch every buffer a chain writes first, and the whole partial area of the GEMM workspace,
holds a NaN sentinel (the page list: page 0, which no sequence owns), so a stale read shows as a NaN or a wrong page, not as a
plausible number. Written buffers sit between guard bands, and the workspace counters must be zero after every launch.

Modes, each against the reference on the same inputs: eager launches (twice, same bits), PDL behind the slow predecessor of
test_gpu_pdl_hazards.py (which stages the next inputs and snapshots every written buffer), and a CUDA graph of the launch
under PDL replayed on three new input versions. The decode step built as a program is compared the same way with the step
recorded with a separator after each persistent op."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from rtp_llm_b200._lib import B200_FMT_INT4, B200_FMT_INT8  # noqa: E402
from rtp_llm_b200.decode_step import LLAMA3_8B, TINY, DecodeStep  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests import pdl_cases  # noqa: E402
from tests import program_chains as pc  # noqa: E402
from tests.test_gpu_pdl_hazards import Writer  # noqa: E402
from tests.test_gpu_program_replay import differing  # noqa: E402

DEV = torch.device("cuda")
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
VERSIONS = (0, 1, 2, 3)          # input versions: 0 eager, 1 behind the slow predecessor, 1..3 graph replays
ROPE_BASE, EPS = 500000.0, 1e-5


def _separator(logits, out, counts):
    ops.argmax(logits, out=out)
    counts.separators += 1


class ChainRun:
    """The device buffers of one chain and its two recordings."""

    def __init__(self, chain: pc.Chain):
        self.chain = c = chain
        dtype = DT[c.dtype]
        g = torch.Generator().manual_seed(11)
        self.static = {}
        for i, op in enumerate(c.ops):
            if op.kind == "gemm":
                self.static[i] = (pdl_cases._weight(op.fmt, dtype, op.K, op.N, g),
                                  pdl_cases._randn(g, op.N, dtype=dtype) if op.bias else None)
            elif op.kind == "norm":
                self.static[i] = (1 + 0.3 * torch.randn(op.hidden, generator=g)).to(dtype).to(DEV)
            elif op.kind == "embed":
                self.static[i] = pdl_cases._randn(g, c.vocab, op.hidden, dtype=dtype)
        self.shapes = pc.shapes(c)
        self.roles = pc.buffer_roles(c)
        self.written = pc.written(c)
        self.bands, self.b = {}, {}
        for name, (shape, kind) in self.shapes.items():
            if name in self.written:
                if kind == "i32":
                    band, v = probe.guarded_empty(shape[:-1] + (2 * shape[-1],), torch.int16)
                    v = v.view(torch.int32)
                else:
                    band, v = probe.guarded_empty(shape, dtype)
                self.bands[name] = band
            else:
                v = torch.empty(shape, dtype=torch.int32 if kind == "i32" else dtype, device=DEV)
            self.b[name] = v
        self.inputs = [k for k, r in self.roles.items() if r == "in"]
        self.versions = {s: self._version(s) for s in VERSIONS}
        gemms = [(op.K, op.N) for op in c.ops if op.kind == "gemm"]
        self.ws = ops.gemm_workspace(c.B, gemms, DEV) if gemms else torch.zeros(pc.SEM_BYTES, dtype=torch.uint8, device=DEV)
        self.attn_ws = ops.attn_workspace(c.B, c.Hq, c.Hkv, c.M * c.T, DEV)
        self.sep_logits = torch.randn(1, 8, generator=g).to(DEV)
        self.sep_out = torch.zeros(1, dtype=torch.int32, device=DEV)

    def _version(self, seed: int) -> dict:
        c, g = self.chain, torch.Generator().manual_seed(1000 + seed)
        d = {}
        for name in self.inputs:
            shape, kind = self.shapes[name]
            if name in ("bid", "pl"):
                bid = (torch.randperm(c.B * c.M, generator=g) + 1).to(torch.int32).view(c.B, c.M)
                d[name] = bid if name == "bid" else torch.stack([2 * bid, 2 * bid + 1], 1).view(c.B, 1, 2, c.M)
            elif name == "seq":
                d[name] = torch.randint(0, c.M * c.T - 1, shape, generator=g, dtype=torch.int32)
            elif name == "ids":
                d[name] = torch.randint(0, c.vocab, shape, generator=g, dtype=torch.int32)
            else:
                d[name] = torch.randn(shape, generator=g).to(DT[c.dtype])
        return {k: v.to(DEV) for k, v in d.items()}

    # ---- recording
    def calls(self, separate: bool, counts: pc.Counts) -> None:
        c, b = self.chain, self.b
        for i, op in enumerate(c.ops):
            if op.kind == "gemm":
                w, bias = self.static[i]
                ops.wo_gemm(b[op.x], w, self.ws, bias=bias, out=b[op.y], silu_mul=op.silu)
            elif op.kind == "norm":
                ops.add_rmsnorm(b[op.x], b[op.res] if op.res else None, self.static[i], EPS, out=b[op.y])
            elif op.kind == "rope":
                ops.rope_append(b[op.x], b["pool"], b["pl"], b["seq"], c.Hq, ROPE_BASE, q_out=b[op.y])
            elif op.kind == "embed":
                ops.embedding(b[op.x], self.static[i], out=b[op.y])
            elif op.kind == "table":
                ops.convert_block_table(b[op.x], out=b[op.y])
            else:
                ops.paged_decode_attn(b[op.x], b["pool"], b["pl"], b["seq"], c.M * c.T, self.attn_ws, out=b[op.y])
            if pc.persistent(op, c.B):
                counts.persistent += 1
                if separate:
                    _separator(self.sep_logits, self.sep_out, counts)
            else:
                counts.plain += 1

    def record(self, separate: bool):
        prog, counts = ops.Program(), pc.Counts()
        with prog.record():
            self.calls(separate, counts)
        return prog, counts

    # ---- one launch
    def reset(self, seed: int) -> None:
        for k in self.inputs:
            self.b[k].copy_(self.versions[seed][k])
        for k in self.written:
            if self.roles[k] == "out":
                v = self.b[k]
                if v.dtype == torch.int32:
                    v.zero_()
                else:
                    v.view(torch.int16).fill_(probe.SENTINEL)
        self.ws[pc.SEM_BYTES:].view(torch.int16).fill_(probe.SENTINEL)

    def checked(self, what: str) -> dict:
        """The written buffers after a launch, once the launch's own invariants hold."""
        torch.cuda.synchronize()
        assert not self.ws[:pc.SEM_BYTES].any(), f"{what}: workspace counters not back to zero"
        pad = probe.GUARD_BYTES // 2
        for k, band in self.bands.items():
            hit = int((band[:pad] != probe.SENTINEL).sum() + (band[band.numel() - pad:] != probe.SENTINEL).sum())
            assert hit == 0, f"{what}: {hit} guard-band elements of {k} overwritten"
        for k in self.written:
            v = self.b[k]
            if self.roles[k] == "out" and v.dtype != torch.int32:
                left = int((v.view(torch.int16) == probe.SENTINEL).sum())
                assert left == 0, f"{what}: {left} elements of {k} still hold the sentinel (never written)"
        return {k: self.b[k].clone() for k in self.written}

    def launch(self, prog, seed: int, what: str) -> dict:
        self.reset(seed)
        prog.launch()
        return self.checked(what)


def _same(got: dict, ref: dict, what: str) -> None:
    bad = differing(got, ref)
    detail = []
    for k in bad:
        g, r = got[k], ref[k]
        if g.dtype == torch.int32:
            detail.append(f"{k}: {int((g != r).sum())} entries differ")
        else:
            gf = g.float()
            detail.append(f"{k}: {int((g.view(torch.int16) != r.view(torch.int16)).sum())} of {g.numel()} differ, "
                          f"{int(torch.isnan(gf).sum())} NaN")
    assert not bad, f"{what}: differs from the separated reference in " + "; ".join(detail)


@pytest.mark.parametrize("chain", pc.CHAINS, ids=[c.name for c in pc.CHAINS])
def test_chain_gives_the_bits_of_its_ops_one_segment_each(chain):
    run = ChainRun(chain)
    ops.set_pdl(False)
    fused, fc = run.record(separate=False)
    ref, rc = run.record(separate=True)
    segs = pc.segments(chain)
    assert fused.num_ops == ref.num_ops == fc.persistent == rc.persistent
    assert fused.num_launches == len(segs), f"recorder made {fused.num_launches} launches, the restated rule {len(segs)}"
    assert ref.num_launches == rc.persistent + rc.separators + rc.plain, "a reference segment holds more than one op"
    assert any(len(s.get("ops", ())) > 1 for s in segs)
    try:
        refs = {s: run.launch(ref, s, f"reference v{s}") for s in VERSIONS}
        assert differing(refs[0], refs[1]), "input versions 0 and 1 give the same bits (vacuous)"
        # eager, twice in a row
        first = run.launch(fused, 0, "eager")
        _same(first, refs[0], "eager")
        again = run.launch(fused, 0, "eager, second launch")
        assert not differing(again, first), "two launches in a row differ"

        # PDL behind the slow predecessor, which stages version 1 over the live inputs
        staged = {k: run.versions[1][k].clone() for k in run.inputs}
        snaps = {k: torch.empty_like(run.b[k]) for k in run.written}
        writer = Writer([(run.b[k], snaps[k]) for k in run.written], [(staged[k], run.b[k]) for k in run.inputs])
        run.reset(0)
        entry = {k: run.b[k].clone() for k in run.written}
        torch.cuda.synchronize()
        ops.set_pdl(True)
        writer.launch()
        fused.launch()
        ops.set_pdl(False)
        got = run.checked("pdl")
        _same(got, refs[1], "behind the slow predecessor (PDL)")
        early = [k for k in run.written if not torch.equal(snaps[k].view(torch.uint8), entry[k].view(torch.uint8))]
        assert not early, f"written before the grid dependency resolved: {early}"

        # graph of the launch under PDL, replayed on new inputs
        run.reset(1)
        torch.cuda.synchronize()
        ops.set_pdl(True)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fused.launch()
        ops.set_pdl(False)
        for s in VERSIONS[1:]:
            run.reset(s)
            graph.replay()
            _same(run.checked(f"graph v{s}"), refs[s], f"graph + PDL replay on version {s}")
    finally:
        ops.set_pdl(False)


# ---------------------------------------------------------------------------------------------- the plan seen on the device
def _split_shapes():
    seen = {}
    for c in pc.CHAINS:
        cov = pc.coverage(c)
        for i, rec in cov["ops"].items():
            op = c.ops[i]
            if rec.get("S", 1) > 1:
                seen.setdefault((op.fmt, c.dtype, c.B, op.K, op.N), rec)
    return sorted(seen.items())


SPLITS = _split_shapes()


@pytest.mark.parametrize("shape,plan", SPLITS, ids=[f"{f} {d} b{B} K{K} N{N}" for (f, d, B, K, N), _ in SPLITS])
def test_a_split_op_writes_exactly_the_partials_of_the_restated_plan(shape, plan):
    fmt, dt, B, K, N = shape
    dtype = DT[dt]
    g = torch.Generator().manual_seed(5)
    w = pdl_cases._weight(fmt, dtype, K, N, g)
    x = pdl_cases._randn(g, B, K, dtype=dtype)
    ws = ops.gemm_workspace(B, [(K, N)], DEV)
    y = torch.empty(B, N, dtype=dtype, device=DEV)
    prog = ops.Program()
    with prog.record():
        ops.wo_gemm(x, w, ws, out=y)
    assert prog.num_ops == 1
    part = ws[pc.SEM_BYTES:].view(torch.int32)
    sentinel = (probe.SENTINEL << 16) | probe.SENTINEL
    part.fill_(sentinel)
    prog.launch()
    torch.cuda.synchronize()
    changed = int((part != sentinel).sum())
    expect = pc.n_tiles(pc.gemm("x", "y", fmt, K, N)) * plan["S"] * pc.bpad_of(B) * pc.TILE_N
    assert changed == expect, f"{changed} fp32 partial words written, the restated plan (S {plan['S']}) gives {expect}"
    assert not ws[:pc.SEM_BYTES].any()


# ---------------------------------------------------------------------------------------------- the decode step
STEPS = {   # name: (config, batch, ctx)
    "tiny int4": (dataclasses.replace(TINY, quant="int4"), 5, 40),
    "tiny int8": (dataclasses.replace(TINY, quant="int8"), 17, 40),
    "Llama-3-8B 2 layers int4 b32": (dataclasses.replace(LLAMA3_8B, layers=2, quant="int4"), 32, 200),
}


def _persistent_call(name, args, kw) -> bool:
    if name == "wo_gemm":
        x, w = args[0], args[1]
        return w.fmt in (B200_FMT_INT4, B200_FMT_INT8) and x.shape[0] <= 64 and w.perm is None
    if name == "add_rmsnorm":
        return args[0].shape[1] <= pc.SEG_NORM_MAX_HIDDEN
    if name == "rope_append":
        return kw.get("q_len", 1) == 1
    return True


def _build_separated(m, monkeypatch) -> pc.Counts:
    """m.build_program() with a separator after every persistent-capable call (the step itself is not changed)."""
    counts = pc.Counts()
    m._sep = (torch.randn(1, 8, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV))
    with monkeypatch.context() as mp:
        for name in ("wo_gemm", "add_rmsnorm", "rope_append", "embedding", "convert_block_table"):
            orig = getattr(ops, name)

            def wrapped(*args, _orig=orig, _name=name, **kw):
                out = _orig(*args, **kw)
                if _persistent_call(_name, args, kw):
                    counts.persistent += 1
                    _separator(*m._sep, counts)
                return out
            mp.setattr(ops, name, wrapped)
        m.build_program()
    return counts


def _step_state(m) -> dict:
    s = dict(logits=m.logits, next_ids=m.next_ids, resid=m.resid, x=m.x, qkv=m.qkv, attn=m.attn, proj=m.proj)
    for i, L in enumerate(m.layers):
        s[f"kv{i}"] = L["kv"]
    return {k: v.detach().clone() for k, v in s.items()}


def _feed(ms, k):
    g = torch.Generator().manual_seed(50 + k)
    ids = torch.randint(0, ms[0].vocab, tuple(ms[0].ids_h.shape), generator=g, dtype=torch.int32)
    for m in ms:
        m.ids_h.copy_(ids)
        m.upload_inputs()


@pytest.mark.parametrize("mode", ["eager", "graph+pdl"])
@pytest.mark.parametrize("name", list(STEPS))
def test_step_program_gives_the_bits_of_its_ops_one_segment_each(name, mode, monkeypatch):
    cfg, batch, ctx = STEPS[name]
    pdl = mode == "graph+pdl"
    try:
        ops.set_pdl(pdl)
        fused = DecodeStep(cfg, batch, ctx, DEV, seed=3, ragged=True, pdl=pdl)
        sep = DecodeStep(cfg, batch, ctx, DEV, seed=3, ragged=True, pdl=pdl)
        n_op = []
        for m in (fused, sep):         # one op-by-op step each: it counts the step's launches and leaves both in one state
            n0 = ops.launch_count()
            m.step()
            n_op.append(ops.launch_count() - n0)
        torch.cuda.synchronize()
        assert n_op[0] == n_op[1]
        fused.build_program()
        counts = _build_separated(sep, monkeypatch)
        assert fused.prog.num_ops == sep.prog.num_ops == counts.persistent
        assert sep.prog.num_launches == n_op[0] + counts.separators, "a reference segment holds more than one op"
        assert fused.prog.num_launches < n_op[0]
        if pdl:
            fused.capture()
            sep.capture()
        for k in range(3):
            for m in (fused, sep):
                ops.set_pdl(pdl)
                m.replay() if pdl else m.run()
            torch.cuda.synchronize()
            a, b = _step_state(fused), _step_state(sep)
            bad = differing(a, b)
            assert not bad, f"step {k}: the program differs from its ops one segment each in {bad}"
            _feed((fused, sep), k)
    finally:
        ops.set_pdl(False)
