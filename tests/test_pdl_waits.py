"""CPU test: every kernel the library may launch with programmatic dependent launch executes griddepcontrol.wait.

Under PDL (b200_set_pdl(1), bench.py's default) a kernel launched through launch_ex may start while the kernel before it
still runs; only griddepcontrol.wait (SASS: ACQBULK) makes that kernel's writes visible. A kernel without it reads stale
inputs, at random, only on the GPU and only with PDL on. Kernels launched with plain <<<>>> carry no PDL attribute and are
exempt; they are listed by name, and the source must launch each of them that way and no other kernel."""
import os
import re
import shutil
import subprocess

import pytest

from rtp_llm_b200 import build

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtp_llm_b200", "csrc")
PLAIN_LAUNCH = {"convert_block_table_kernel", "paged_attn_plan_kernel", "embedding_kernel", "argmax_kernel", "pack_w4_kernel",
                "pack_w8_kernel", "pack_w8g_kernel"}


def _source(pattern):
    return {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if re.fullmatch(pattern, f)}


def _kernels_defined():
    names = set()
    for src in _source(r".*\.(cuh|cu)").values():
        names |= set(re.findall(r"__global__[^;{]*?\b(\w+_kernel)\s*\(", src))
    return names


def _sass_by_kernel(defined):
    """{kernel name: [SASS of each instantiation]}, every function of the library matched to the kernel it instantiates."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", build.build()], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", sass)
    out = {}
    for mangled, body in zip(parts[1::2], parts[2::2]):
        hits = [k for k in defined if f"{len(k)}{k}" in mangled]          # Itanium mangling: <length><identifier>
        assert len(hits) == 1, f"{mangled}: matches {hits} of the kernels defined in csrc/"
        out.setdefault(hits[0], []).append(body)
    return out


def test_plain_launches_are_exactly_the_exempt_kernels():
    launches = "".join(_source(r"c_api\.cu|.*_inst\.cuh").values())
    plain = set(re.findall(r"\b(\w+_kernel)\s*(?:<[^<>;]*>)?\s*<<<", launches))
    assert plain == PLAIN_LAUNCH
    assert not PLAIN_LAUNCH & set(re.findall(r"launch_ex\(\s*(\w+)", launches))


def test_every_kernel_launched_with_pdl_waits_for_its_predecessor():
    defined = _kernels_defined()
    assert PLAIN_LAUNCH <= defined and "sample_kernel" in defined and "wo_gemm_kernel" in defined
    by_kernel = _sass_by_kernel(defined)
    assert set(by_kernel) == defined, f"kernels missing from the library: {defined - set(by_kernel)}"
    missing = sorted(k for k, bodies in by_kernel.items() if k not in PLAIN_LAUNCH and not all("ACQBULK" in b for b in bodies))
    assert not missing, f"launched through launch_ex (PDL) without griddepcontrol.wait: {missing}"
