"""CPU test: libb200_decode.so loads and exports every symbol include/b200_decode_ops.h declares (no compute calls)."""
import ctypes
import os
import re

from rtp_llm_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b200_decode_ops.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    path = build.build()
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 19
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    # and the ctypes signature table covers exactly the header
    assert sorted(_lib.SIGNATURES) == names


def test_argument_errors_are_reported_not_crashed():
    lib = _lib.load()
    # null pointers / bad shapes are rejected on the host before any CUDA call
    assert lib.b200_convert_block_table(None, None, 4, 8, None) == -1
    assert b"null" in lib.b200_last_error()
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4, 100, 64) == 0          # K not a multiple of 128
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT4, 256, 256) == 2 * 2 * 8704
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT8, 256, 200) == 2 * 2 * 16384   # N padded to 128-feature tiles
    assert lib.b200_paged_decode_attn_workspace_bytes(32, 32, 8, 2048) > 0
    assert lib.b200_wo_gemm_workspace_bytes(32, 4096, 4096) >= 16384


def test_argument_errors_of_the_round2_entry_points():
    """Validation happens on the host before any CUDA call: checkable without a GPU. Mirrors the reference ops' behaviour of
    raising on bad shapes (XQAAttnOp.cc:62-70 RTP_LLM_CHECK_WITH_INFO) instead of launching."""
    import ctypes
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    regs = (ctypes.c_void_p * 8)(*([p.value] * 8))
    # 8-bit group-wise blobs: 16384 payload bytes + 512 bytes of scales / zero*scale per (128 x 128) block
    assert lib.b200_wo_gemm_packed_bytes(_lib.B200_FMT_INT8G, 256, 256) == 2 * 2 * 16896
    assert lib.b200_wo_gemm_packed_bytes(7, 256, 256) == 0                                    # unknown format
    assert lib.b200_pack_w8g(p, p, p, 256, 256, 64, p, None) == -1 and b"group" in lib.b200_last_error()
    assert lib.b200_pack_w8g(p, p, p, 100, 256, 128, p, None) == -1 and b"multiple of 128" in lib.b200_last_error()
    # GEMM + reduce-scatter: world / shape limits
    args = (_lib.B200_FMT_INT4, 0, p, 32, 512, 4096, p, None, None, p, p, 4096, 0)
    assert lib.b200_wo_gemm_rs(*args, regs, 1 << 19, 0, 1, None) == -1 and b"rank/world" in lib.b200_last_error()
    assert lib.b200_wo_gemm_rs(*args, regs, 1 << 10, 0, 2, None) == -1 and b"exceeds the region" in lib.b200_last_error()
    bad_n = (_lib.B200_FMT_INT4, 0, p, 32, 512, 4160, p, None, None, p, p, 4096, 0)
    assert lib.b200_wo_gemm_rs(*bad_n, regs, 1 << 19, 0, 2, None) == -1 and b"multiple of 128" in lib.b200_last_error()
    silu = args[:-1] + (_lib.B200_GEMM_SILU_MUL,)
    assert lib.b200_wo_gemm_rs(*silu, regs, 1 << 19, 0, 2, None) == -1 and b"SILU_MUL" in lib.b200_last_error()
    assert lib.b200_wo_gemm(9, 0, p, 32, 512, 4096, p, None, None, p, p, 4096, 0, None) == -1 and b"unknown weight format" in lib.b200_last_error()
    assert lib.b200_wo_gemm(_lib.B200_FMT_INT8, 0, p, 32, 512, 4096, p, None, None, p, p, 4096, 0, None) == -1 and b"col_scale" in lib.b200_last_error()
    # the second half of the exchange shares the all-reduce+norm checks
    assert lib.b200_peer_gather_norm(p, p, p, p, 0, 32, 4100, 1e-5, regs, 1 << 19, 0, 2, None) == -1 and b"hidden" in lib.b200_last_error()


def test_sass_uses_the_hopper_paths():
    """The built library must contain warpgroup MMA (wgmma) and TMA instructions: tensor-map loads and bulk copies."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", build.build()], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "WARPGROUP.ARRIVE", "UTMALDG", "UBLKCP"):
        assert mnem in sass, mnem


def test_launch_shape_heuristics_on_the_baseline_shapes():
    """Host-only: the split choices of the launch-shape heuristics on the baseline shapes (132 SMs when no device is visible)."""
    import ctypes
    lib = _lib.load()

    def attn(units, seq):
        ns, c = ctypes.c_int(), ctypes.c_int()
        assert lib.b200_plan_attn_split(units, seq, ctypes.byref(ns), ctypes.byref(c)) == 0
        return ns.value, c.value

    def gemm(K, N):
        ns, kb = ctypes.c_int(), ctypes.c_int()
        assert lib.b200_plan_gemm_split(K, N, ctypes.byref(ns), ctypes.byref(kb)) == 0
        return ns.value, kb.value
    assert attn(32 * 8, 2048) == (1, 32)          # Llama-3-8B B32 ctx2048: one CTA per (sequence, kv head)
    assert attn(32 * 4, 2048) == (1, 32)          # TP2 per-rank shape
    assert attn(32 * 1, 2048) == (2, 16)          # TP8 per-rank shape: 32 units, the sequence split in two (the H100 cost
                                                  # model's choice; not measured against other splits on an H100)
    ns, c = attn(8, 4096)                          # batch 1: split the sequence to fill the GPU
    assert ns > 1 and ns * c >= 64
    assert gemm(4096, 28672) == (1, 32)           # w13: 224 tiles, no split
    ns, kb = gemm(4096, 4096)                     # o-proj: 32 tiles -> cluster of 8 along k
    assert ns == 8 and kb == 4
    ns, kb = gemm(4096, 6144)                     # qkv: 48 tiles -> cluster of 4
    assert ns == 4 and kb == 8
    assert gemm(4096, 128256)[0] == 1             # lm_head: > one wave of tiles, never split
    assert lib.b200_plan_gemm_split(100, 64, None, None) == -1
