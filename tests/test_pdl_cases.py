"""CPU test: the PDL hazard harness (test_gpu_pdl_hazards.py) has a case for every kernel the library launches through launch_ex.

A kernel launched with the PDL attribute may start while its predecessor still runs; the harness checks, kernel by kernel,
that nothing is read or written before griddepcontrol.wait. A new PDL kernel must get a case there, or the harness would
never see it. The peer collectives poll memory that other ranks write and are tested rank by rank elsewhere; the plainly
launched kernels (test_pdl_waits.PLAIN_LAUNCH) carry no PDL attribute."""
import re

from tests.pdl_cases import CASES
from tests.test_pdl_waits import PLAIN_LAUNCH, _kernels_defined, _source

PEER_KERNELS = {"peer_allreduce_kernel", "peer_allreduce_twoshot_kernel", "peer_allreduce_norm_kernel", "peer_argmax_kernel"}


def _pdl_kernels():
    """Every kernel name an op hands to launch_op / launch_or_record (the names a launch is recorded under), less the plain
    launches, plus "wo_gemm_kernel/rs" when a translation unit instantiates the reduce-scatter GEMM (B200_GEMM_VAR 1): it is
    launched under the plain GEMM's name but has its own epilogue and writes into the peer regions."""
    launches = "".join(_source(r"c_api\.cu|.*_inst\.cuh").values())
    names = set(re.findall(r'"(\w+_kernel)"', launches)) - PLAIN_LAUNCH
    if any(re.search(r"#define\s+B200_GEMM_VAR\s+1\b", src) for src in _source(r"gemm_cluster.*\.cu").values()):
        names.add("wo_gemm_kernel/rs")
    return names


def test_every_pdl_kernel_has_a_hazard_case():
    pdl = _pdl_kernels()
    assert pdl - {"wo_gemm_kernel/rs"} <= _kernels_defined(), f"launch names that are no kernel of csrc/: {pdl - _kernels_defined()}"
    assert {"wo_gemm_kernel", "wo_gemm_kernel/rs", "decode_segment_kernel", "paged_decode_attn_kernel"} <= pdl
    covered = {k for c in CASES for k in c.kernels}
    missing = sorted(pdl - covered - PEER_KERNELS)
    assert not missing, f"PDL kernels without a case in tests/pdl_cases.py: {missing}"
    assert PEER_KERNELS <= pdl, f"peer kernels no longer launched: {PEER_KERNELS - pdl}"
    assert covered <= pdl, f"cases name kernels the library does not launch with PDL: {covered - pdl}"


def test_case_names_are_unique():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))
