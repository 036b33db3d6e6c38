"""CPU tests of the rope config at the attention seams: the cos/sin table builder against the reference-built golden rows, which
kernel entry each rope style takes, which configs the seams refuse, the new C ABI entry's argument checks and the pybind
RopeConfig surface."""
import ctypes
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rtp_llm_b200 import _lib, attention, build, ops, rope

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", ["rope_cache_base_scale2", "rope_cache_yarn"])
def test_table_builder_reproduces_the_reference_rows_bit_for_bit(name):
    g = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    cfg = {k[4:]: (float(g[k]) if g[k].dtype.kind == "f" else int(g[k])) for k in g.files if k.startswith("cfg_")}
    spec = rope.spec_of(SimpleNamespace(**cfg), int(g["head_dim"]))
    table = rope.build_table(spec)
    assert table.dtype == torch.float32 and table.shape == (int(g["cache_positions"]), cfg["dim"])
    rows = table.numpy()[g["positions"]]
    assert np.array_equal(rows.view(np.uint32), np.ascontiguousarray(g["cache_rows"], np.float32).view(np.uint32))


def test_table_is_built_only_for_base_and_yarn_with_positions():
    base = dict(style=rope.BASE, dim=64, base=10000.0, scale=2.0, max_pos=100)
    assert rope.build_table(rope.RopeSpec(**base)).shape == (200, 64)
    for style in (rope.NO, rope.DYNAMIC_NTK, rope.QWEN_DYNAMIC_NTK, rope.LLAMA3):
        assert rope.build_table(rope.RopeSpec(**dict(base, style=style))) is None
    assert rope.build_table(rope.RopeSpec(**dict(base, max_pos=0))) is None
    dev = torch.device("cpu")
    assert rope.table(rope.RopeSpec(**base), dev) is rope.table(rope.RopeSpec(**base), dev)     # built once per config


D, HQ, HKV = 128, 4, 2
LLAMA31 = dict(style=6, base=500000.0, scale=8.0, factor1=1.0, factor2=4.0, max_pos=8192)
YARN = dict(style=5, base=1000000.0, scale=4.0, factor1=1.0, factor2=32.0, max_pos=32768, mscale=1.1)
# name, rope_config fields (None: no rope_config at all), use_logn_attn, position ids, expected path (None: refused)
PATHS = [
    ("no rope_config", None, False, False, "plain"),
    ("base only", dict(base=500000.0), False, False, "plain"),
    ("base style 1 full dim", dict(style=1, dim=D, base=10000.0, scale=1.0), False, False, "plain"),
    ("base dim 0", dict(style=1, dim=0, base=10000.0), False, False, "plain"),
    ("base + logn", dict(style=1, base=10000.0, max_pos=2048), True, False, "ex+table"),
    ("base + position ids", dict(style=1, base=10000.0, max_pos=2048), False, True, "ex+table"),
    ("base linear scale", dict(style=1, base=10000.0, scale=4.0, max_pos=2048), False, False, "ex+table"),
    ("base partial dim", dict(style=1, dim=64, base=10000.0, max_pos=2048), False, False, "ex+table"),
    ("llama3", LLAMA31, False, False, "ex"),
    ("yarn", YARN, False, False, "ex+table"),
    ("dynamic ntk", dict(style=3, base=10000.0, scale=2.0, max_pos=512), False, False, "ex"),
    ("qwen dynamic ntk", dict(style=4, base=10000.0, max_pos=512), False, True, "ex"),
    ("no rotation", dict(style=0), False, False, "ex"),
    ("glm2", dict(style=2, base=10000.0), False, False, None),
    ("mrope", dict(style=7, base=10000.0), False, False, None),
    ("unknown style", dict(style=9, base=10000.0), False, False, None),
    ("not neox", dict(style=1, base=10000.0, is_neox_style=False), False, False, None),
    ("odd dim", dict(style=1, dim=63, base=10000.0), False, False, None),
    ("dim above head", dict(style=1, dim=2 * D, base=10000.0), False, False, None),
    ("base <= 1", dict(style=6, base=1.0), False, False, None),
]


def _attn_cfg(fields, logn):
    cfg = SimpleNamespace(head_num=HQ, kv_head_num=HKV, size_per_head=D, tokens_per_block=16, need_rope_kv_cache=True)
    if fields is not None:
        cfg.rope_config = SimpleNamespace(**fields)
    if logn:
        cfg.use_logn_attn = True
    return cfg


@pytest.mark.parametrize("q_len", [1, 3])
@pytest.mark.parametrize("case", PATHS, ids=[c[0] for c in PATHS])
def test_seam_selects_the_kernel_entry_per_rope_config(case, q_len, monkeypatch):
    name, fields, logn, with_pid, want = case
    op = attention.B200RopeKVCacheDecodeOp(_attn_cfg(fields, logn))
    assert op.supported() == (want is not None)
    if want is None:
        assert not attention.B200DecodeImpl.support(_attn_cfg(fields, logn), SimpleNamespace(is_prefill=False))
        return
    calls = []
    monkeypatch.setattr(ops, "rope_append", lambda *a, **k: calls.append(("plain", a, k)))
    monkeypatch.setattr(ops, "rope_append_ex", lambda *a, **k: calls.append(("ex", a, k)))
    B = 2
    qkv = torch.zeros(B * q_len, (HQ + 2 * HKV) * D, dtype=torch.float16)
    pool = torch.zeros(3, 2, HKV, 16, D, dtype=torch.float16)
    pl, seq = torch.zeros(B, 1, 2, 1, dtype=torch.int32), torch.zeros(B, dtype=torch.int32)
    pid = torch.arange(B * q_len, dtype=torch.int32) if with_pid else None
    op.forward(qkv, pool, pl, seq, q_len, pid)
    (kind, args, kw), = calls
    assert kw["q_len"] == q_len
    if want == "plain":
        assert kind == "plain" and args[5] == float((fields or {}).get("base", 10000.0))
        return
    assert kind == "ex"
    c = args[5]
    spec = rope.spec_of(SimpleNamespace(**fields), D)
    assert (c.style, c.dim, c.max_pos) == (spec.style, spec.dim, spec.max_pos)
    assert np.float32(c.base) == np.float32(spec.base) and np.float32(c.scale) == np.float32(spec.scale)
    assert kw["use_logn_attn"] == logn
    assert (kw["position_ids"] is not None) == with_pid
    table = kw["cos_sin_cache"]
    assert (table is not None) == (want == "ex+table")
    if table is not None:
        assert table.shape == (int(spec.max_pos * spec.scale), spec.dim)


def test_llama31_config_fields_reach_the_kernel_config():
    c = rope.c_config(rope.spec_of(SimpleNamespace(**LLAMA31), D))
    assert (c.style, c.dim, c.base, c.scale, c.factor1, c.factor2, c.max_pos) == (6, D, 500000.0, 8.0, 1.0, 4.0, 8192)


def test_rope_append_ex_multi_argument_checks():
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = _lib.RopeConfig(style=1, dim=128, base=10000.0, scale=1.0, factor1=1.0, factor2=1.0, max_pos=2048, extrapolation_factor=1.0,
                         mscale=1.0)
    cfg = ctypes.cast(ctypes.pointer(rc), ctypes.c_void_p)
    args = lambda q_len, qkv=p: (qkv, None, p, p, p, p, None, None, 0, cfg, 0, 0, 2, 4, 2, 128, 4, 16, q_len, None)
    assert lib.b200_rope_append_ex_multi(*args(0)) == -1 and b"q_len" in lib.b200_last_error()
    assert lib.b200_rope_append_ex_multi(*args(2, None)) == -1 and b"null" in lib.b200_last_error()
    rc.dim = 130
    assert lib.b200_rope_append_ex_multi(*args(2)) == -1 and b"rotary dim" in lib.b200_last_error()


def _pybind():
    spec = importlib.util.spec_from_file_location("b200_compute_ops", build.build_pybind())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.rtp_llm_ops


def test_pybind_rope_config_mirrors_the_reference_fields_with_base_defaults():
    m = _pybind()
    r = m.RopeConfig()
    assert (r.style, r.dim, r.base, r.scale, r.max_pos, r.is_neox_style) == (1, 0, 10000.0, 1.0, 0, True)
    for k, v in dict(LLAMA31, dim=64, extrapolation_factor=1.0, mscale=1.1, is_neox_style=False).items():
        setattr(r, k, v)
        assert getattr(r, k) == pytest.approx(v)
    cfg = m.AttentionConfigs()
    assert cfg.use_logn_attn is False
    cfg.rope_config = r
    assert cfg.rope_config.style == 6
    inp = m.PyAttentionInputs()
    inp.input_lengths = torch.tensor([3, 3], dtype=torch.int32)
    inp.combo_position_ids = torch.arange(6, dtype=torch.int32)
    assert inp.combo_position_ids.numel() == 6
    assert hasattr(m.B200AttnParams, "q_len")
