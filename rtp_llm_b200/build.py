"""Build libb200_decode.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc. No JIT cache: the library is built
once, next to its sources, and loaded from there."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200_decode.so")
# translation units compile in parallel (the persistent-kernel instantiations dominate the build time)
SOURCES = ["c_api.cu", "gemm_cluster.cu", "gemm_cluster_rs.cu", "segment_f16.cu", "segment_bf16.cu"]
NVCC_FLAGS = ["-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
              "-Xcompiler", "-fPIC", "-DB200_BUILD"]
TESTREF_SRC = os.path.join(ROOT, "tests", "native", "test_ref.cu")
TESTREF_LIB = os.path.join(ROOT, "tests", "native", "libb200_testref.so")


def _deps():
    """Every header of csrc/ plus the public header: an edited kernel can never run against a stale library."""
    hdr = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    return hdr + [os.path.join(ROOT, "include", "b200_decode_ops.h"), os.path.abspath(__file__)]


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _stale() -> bool:
    return _newer(LIB, _deps() + [os.path.join(CSRC, s) for s in SOURCES])


STAMP = LIB + ".stamp"


def source_digest() -> str:
    """sha256 over every source / header / flag the library is built from. build() records it next to the .so; _lib.load()
    compares it, so an edited kernel can never run against an old library -- by CONTENT, because file times do not survive
    the copy to the GPU box."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for p in sorted(_deps()[:-1] + [os.path.join(CSRC, s) for s in SOURCES]):     # (build.py itself is not an input of nvcc)
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def stamp_matches() -> bool:
    """True when the library on disk was built from the sources on disk (or carries no stamp: a library of unknown origin
    is used as it is, as before)."""
    if not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() == source_digest()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale() and stamp_matches():
        if not os.path.exists(STAMP):
            with open(STAMP, "w") as f:
                f.write(source_digest())
        return LIB
    from concurrent.futures import ThreadPoolExecutor
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJDIR, exist_ok=True)
    hdrs = _deps()

    def compile_one(src):
        obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        path = os.path.join(CSRC, src)
        if force or _newer(obj, hdrs + [path]):
            subprocess.check_call([nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", path, "-o", obj])
        return obj
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    subprocess.check_call([nvcc, "-shared", "-o", LIB + ".tmp"] + objs + ["-lcudart"])
    os.replace(LIB + ".tmp", LIB)             # atomic: another process never maps a half-written library
    with open(STAMP, "w") as f:
        f.write(source_digest())
    return LIB


def build_testref(force: bool = False) -> str:
    """tests/native/libb200_testref.so: naive CUDA-core checkers used by the GPU tests only (not part of the product)."""
    if not force and not _newer(TESTREF_LIB, [TESTREF_SRC, os.path.join(CSRC, "ptx.cuh")]):
        return TESTREF_LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-shared", "-Xcompiler", "-fPIC",
                           "-o", TESTREF_LIB, TESTREF_SRC, "-lcudart"])
    return TESTREF_LIB


PYBIND_SO = os.path.join(HERE, "b200_compute_ops.so")


def build_pybind(force: bool = False) -> str:
    """Compile csrc/pybind_ops.cc (registerPyModuleOps + the XQAAttnOp-shaped class) against torch's headers and link it to
    libb200_decode.so. Plain g++ (no JIT cache): the .so stays in-tree and travels with the snapshot."""
    src = os.path.join(CSRC, "pybind_ops.cc")
    if not force and os.path.exists(PYBIND_SO) and os.path.getmtime(PYBIND_SO) > max(
            os.path.getmtime(src), os.path.getmtime(os.path.join(HERE, "..", "include", "b200_decode_ops.h"))):
        return PYBIND_SO
    build()
    import sysconfig
    import torch
    from torch.utils import cpp_extension as ce
    inc = ce.include_paths() + [sysconfig.get_paths()["include"], "/usr/local/cuda/include"]
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden", "-DTORCH_EXTENSION_NAME=b200_compute_ops", "-DTORCH_API_INCLUDE_EXTENSION_H",
           f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"] + [f"-I{i}" for i in inc] + \
          [src, "-o", PYBIND_SO, f"-L{libdir}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
           f"-L{HERE}", "-l:libb200_decode.so", "-L/usr/local/cuda/lib64", "-lcudart",
           f"-Wl,-rpath,{libdir}", "-Wl,-rpath,$ORIGIN", "-Wl,-rpath,/usr/local/cuda/lib64"]
    subprocess.check_call(cmd)
    return PYBIND_SO


if __name__ == "__main__":
    if "--pybind" in sys.argv:
        print(build_pybind(force="--force" in sys.argv))
        sys.exit(0)
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
