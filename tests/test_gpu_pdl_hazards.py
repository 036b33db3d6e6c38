"""GPU tests (H100) of every kernel's grid-dependency contract under programmatic dependent launch (PDL).

Under PDL a kernel may be resident while the kernel before it still runs; only its griddepcontrol.wait makes that kernel's
writes visible. Each kernel may read data that is constant after load (weights, gammas, perm, rope tables) before the wait,
and nothing else, and may write nothing before it (DESIGN section 3.4).

The harness puts a slow predecessor in front of each entry point: a writer kernel (tests/native/test_ref.cu), launched
without the PDL attribute, that lets dependents launch, spins for DELAY_NS, snapshots every buffer the entry point writes, and
then copies a staged second version B of every dynamic input over the live inputs, which hold version A. The entry point is
launched right behind it with PDL on. A read before the wait sees A (or the seeded random bytes of an output), so a written
buffer differs from the eager reference on B; a write before the wait shows in the writer's snapshot. A probe kernel first
shows, per resource class, that a dependent does become resident inside the writer's window on this device; the controls
show that the harness catches a load and a store placed before the wait. Each case also runs as a CUDA graph replayed on
three new staged inputs.

Out of scope: the peer collectives (peer_allreduce*, peer_allreduce_norm, peer_argmax), which poll memory other ranks write
(putting a slow writer into their rank-alone harness is its own change), and the kernels of test_pdl_waits.PLAIN_LAUNCH, which
are launched without the PDL attribute."""
from typing import Optional

import pytest
import torch

pytestmark = pytest.mark.gpu

from rtp_llm_b200 import ops  # noqa: E402
from tests import gpu_probe as probe  # noqa: E402
from tests import ref_kernels  # noqa: E402
from tests.pdl_cases import CASES, Case, Spec  # noqa: E402

DEV = torch.device("cuda")
DELAY_NS = 200_000
GRAPH_SEEDS = (1, 2, 3)          # B1, B2, B3; A is seed 0


def _bytes(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().view(-1).view(torch.uint8)


class Writer:
    """The slow predecessor: snapshot ranges (written buffer -> snapshot) then staging ranges (staged input -> live input)."""

    def __init__(self, snaps, stages, delay_ns=DELAY_NS):
        rows = [(s.data_ptr(), d.data_ptr(), s.numel() * s.element_size()) for s, d in list(snaps) + list(stages)]
        for (s, d), n in zip(list(snaps) + list(stages), (r[2] for r in rows)):
            assert d.numel() * d.element_size() == n
        self.copies = torch.tensor(rows or [(0, 0, 0)], dtype=torch.int64, device=DEV)
        self.n_snap, self.n_stage, self.delay = len(snaps), len(stages), delay_ns
        self.times = torch.zeros(2, dtype=torch.int64, device=DEV)

    def launch(self):
        ref_kernels.pdl_writer(self.copies, self.n_snap, self.n_stage, self.delay, self.times)


def _fill(t: torch.Tensor, seed: int) -> None:
    g = torch.Generator().manual_seed(seed)
    _bytes(t).copy_(torch.randint(0, 256, (t.numel() * t.element_size(),), generator=g, dtype=torch.uint8))


class Harness:
    """Live buffers of one case: dynamic inputs (version A at entry), outputs (seeded random bytes at entry), workspaces (zero
    at entry), and the staged inputs and snapshots the writer copies."""

    def __init__(self, case: Case):
        self.case = case
        with probe.env_set(case.env):
            self.spec = spec = case.setup()
            self.versions = {s: spec.dyn(s) for s in (0,) + GRAPH_SEEDS}
        self.live = {k: v.clone() for k, v in self.versions[0].items()}
        self.outs = {k: torch.empty(shape, dtype=dt, device=DEV) for k, (shape, dt) in spec.outs.items()}
        self.ws = {k: torch.zeros(n, dtype=torch.uint8, device=DEV) for k, (n, _) in spec.ws.items()}
        self.bufs = {**spec.static, **self.live, **self.outs, **self.ws}
        self.written = {k: self.bufs[k] for k in list(spec.inplace) + list(self.outs) + list(self.ws)}
        self.staged = {k: v.clone() for k, v in self.live.items()}
        self.snaps = {k: torch.empty_like(v) for k, v in self.written.items()}
        self.writer = Writer([(v, self.snaps[k]) for k, v in self.written.items()],
                             [(self.staged[k], v) for k, v in self.live.items()])

    def reset(self, stage_seed: Optional[int] = None):
        for k, v in self.live.items():
            v.copy_(self.versions[0][k])
        for i, (k, v) in enumerate(self.outs.items()):
            _fill(v, 1000 + i)
        for v in self.ws.values():
            v.zero_()
        if stage_seed is not None:
            for k, v in self.staged.items():
                v.copy_(self.versions[stage_seed][k])
        for v in self.snaps.values():
            v.zero_()
        self.entry = {k: v.clone() for k, v in self.written.items()}

    def call(self):
        with probe.env_set(self.case.env):
            self.spec.call(self.bufs)

    def reference(self, seed: int) -> dict:
        """The written buffers after an eager call on version `seed`, PDL off, from the entry state of a hazard run."""
        self.reset()
        for k, v in self.live.items():
            v.copy_(self.versions[seed][k])
        self.entry = {k: v.clone() for k, v in self.written.items()}
        ops.set_pdl(False)
        self.call()
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in self.written.items()}

    def failures(self, ref: dict, ref_a: dict) -> list:
        """What the harness's own check reports: written buffers that differ from the reference on the staged inputs (a read
        before the wait), snapshots that differ from the entry bytes (a write before the wait), and counters not back to zero."""
        bad = []
        for k, v in self.written.items():
            got, exp = _bytes(v), _bytes(ref[k])
            diff = got != exp
            if diff.any():
                n = int(diff.sum())
                from_a = int((got[diff] == _bytes(ref_a[k])[diff]).sum())
                from_entry = int((got[diff] == _bytes(self.entry[k])[diff]).sum())
                bad.append(f"{k}: {n} bytes differ from the reference on the staged inputs ({from_a} hold the result on the "
                           f"entry inputs A, {from_entry} the entry bytes): read before the grid dependency")
            snap_diff = _bytes(self.snaps[k]) != _bytes(self.entry[k])
            if snap_diff.any():
                bad.append(f"{k}: {int(snap_diff.sum())} bytes written before the grid dependency resolved")
        for k, (_, counters) in self.spec.ws.items():
            if counters and _bytes(self.ws[k])[:counters].any():
                bad.append(f"{k}: counters not back to zero")
        if bad:
            t0, t1 = self.writer.times.tolist()
            bad.append(f"writer copied from {t0} to {t1} ns (globaltimer)")
        return bad


def _run_case(case: Case) -> None:
    h = Harness(case)
    refs = {s: h.reference(s) for s in (0,) + GRAPH_SEEDS}
    differs = [k for k in h.written if not torch.equal(_bytes(refs[0][k]), _bytes(refs[1][k]))]
    assert differs, f"{case.name}: versions A and B give the same bits in every written buffer (vacuous case)"
    try:
        if case.stream:
            h.reset(GRAPH_SEEDS[0])
            torch.cuda.synchronize()
            ops.set_pdl(True)
            torch.cuda.set_sync_debug_mode("error")    # a host synchronisation would let the writer finish first
            try:
                h.writer.launch()
                n0 = ops.launch_count()
                h.call()
                # one library launch per kernel the case names, so nothing of the library's sits between the writer and
                # the PDL kernel; a torch kernel (a memset of an output the call allocates) would not be counted: calls
                # take every buffer preallocated
                assert ops.launch_count() - n0 == len(case.kernels), f"{case.name}: unexpected launches"
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            bad = h.failures(refs[GRAPH_SEEDS[0]], refs[0])
            assert not bad, f"{case.name} (stream): " + "; ".join(bad)
        ops.set_pdl(True)
        h.reset(GRAPH_SEEDS[0])
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            h.writer.launch()
            h.call()
        ops.set_pdl(False)
        for s in GRAPH_SEEDS:
            h.reset(s)
            graph.replay()
            torch.cuda.synchronize()
            bad = h.failures(refs[s], refs[0])
            assert not bad, f"{case.name} (graph, B{s}): " + "; ".join(bad)
    finally:
        ops.set_pdl(False)


# ---------------------------------------------------------------------------------------------- the harness's self-test
def _control(mode: int, graph: bool) -> list:
    n = 1 << 16
    g = torch.Generator().manual_seed(mode)
    versions = {s: torch.randint(-2 ** 31, 2 ** 31 - 1, (n,), generator=g, dtype=torch.int32).to(DEV) for s in (0, 1)}

    def call(b):
        ref_kernels.pdl_copy(b["in"], b["out"], mode)
    spec = Spec(dyn=lambda s: {"in": versions[min(s, 1)].clone()}, call=call, outs={"out": ((n,), torch.int32)})
    case = Case(f"control mode {mode}", (), lambda: spec)
    h = Harness(case)
    ref, ref_a = {"out": versions[1]}, {"out": versions[0]}
    h.reset(1)
    torch.cuda.synchronize()
    if graph:
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            h.writer.launch()
            h.call()
        h.reset(1)
        cg.replay()
    else:
        h.writer.launch()
        h.call()
    torch.cuda.synchronize()
    return h.failures(ref, ref_a)


@pytest.mark.parametrize("graph", [False, True], ids=["stream", "graph"])
def test_controls_pass_a_waiting_copy_and_fail_an_early_load_and_an_early_store(graph):
    assert _control(0, graph) == []
    early_load = _control(1, graph)
    assert early_load and "read before the grid dependency" in early_load[0], early_load
    early_store = _control(2, graph)
    assert any("written before the grid dependency" in f for f in early_store), early_store


# ---------------------------------------------------------------------------------------------- early entry per resource class
def _sms() -> int:
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _attn_smem(D):
    """attn_smem_bytes(D) of csrc/paged_decode_attn.cuh: 3 stages of D / 64 K and V halves of 8 KB, plus 1792 bytes."""
    return 3 * 2 * (D // 64) * 64 * 128 + 1024 + 256 + 512


# The footprints of the library's PDL kernels (threads and dynamic shared memory as csrc/ sets them: kAttnThreads 160,
# gemm_threads() and kSegThreads 320, the GEMM's 106 KB two-per-SM and 216 KB one-per-SM budgets). They are mirrored here,
# not read from the library: a kernel whose footprint grows past its class needs its class updated with it.
RESOURCE_CLASSES = {   # name: (grid x, grid y, threads, dynamic shared memory, cluster x)
    "glue": (lambda: (64, 1, 256, 0, 1)),
    "attention cluster of 8": (lambda: (8, 16, 160, _attn_smem(128), 8)),
    "attention d256 one per SM": (lambda: (4, 32, 160, _attn_smem(256), 1)),
    "gemm 106 KB": (lambda: (2 * _sms(), 1, 320, 106 * 1024, 1)),
    "gemm 216 KB": (lambda: (_sms(), 1, 320, 216 * 1024, 1)),
    "persistent 2 per SM": (lambda: (2 * _sms(), 1, 320, 106 * 1024, 1)),
}


@pytest.mark.parametrize("graph", [False, True], ids=["stream", "graph"])
@pytest.mark.parametrize("cls", list(RESOURCE_CLASSES))
def test_a_dependent_enters_inside_the_writers_window(cls, graph):
    gx, gy, threads, smem, cluster = RESOURCE_CLASSES[cls]()
    entry = torch.zeros(gx * gy, dtype=torch.int64, device=DEV)
    w = Writer([], [])

    def launch():
        w.launch()
        ref_kernels.pdl_probe(gx, gy, threads, smem, cluster, entry)
    launch()                     # the first launch of a kernel loads its module, which holds the launch back
    torch.cuda.synchronize()
    if graph:
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            launch()
        cg.replay()
    else:
        launch()
    torch.cuda.synchronize()
    t0 = int(w.times[0])
    first = int(entry.min())
    early = int((entry < t0).sum())
    print(f"PDL-PROBE {cls} {'graph' if graph else 'stream'}: first CTA entered {(t0 - first) / 1e3:.1f} us before the writer's "
          f"copy; {early} of {entry.numel()} CTAs before it")
    assert first > 0 and first < t0, f"{cls}: no CTA became resident before the writer's copy (first {first}, copy {t0})"


# ---------------------------------------------------------------------------------------------- one case per entry point
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_entry_point_waits_for_its_grid_dependency(case):
    _run_case(case)
