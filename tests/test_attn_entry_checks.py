"""CPU tests of the six paged-attention entries' argument checks: every rejection each entry makes, one bad argument at a time
(status -1 and the message that names it), and what each entry returns for an empty call that also carries one bad argument.
Each call breaks at least one check, so none of them reaches a launch. The mode checks that test_beam_attn.py, test_spec_verify.py
and test_spec_tree.py already make are not repeated here."""
import ctypes

import pytest

from rtp_llm_b200 import _lib

_BUF = (ctypes.c_uint8 * (1 << 16))()
P = (ctypes.addressof(_BUF) + 255) & ~255            # a 256-byte aligned host address: never read, every call is rejected first
ENTRIES = ["plain", "multi", "rope", "beam", "prefix", "tree"]
# a call every check accepts: group 4, 2 query slots per CTA (q_len, beams or chunk members), 2 sequences / requests / chunks
GOOD = dict(q=P, out=P, Hq=8, Hkv=2, D=128, batch=2, slots=2, chunks=2, M=4, max_seq_len=256, T=64, kv=P, page_list=P,
            seq_lens=P, extra=P, offsets=P, rows=P, rope_base=10000.0, ws=P, ws_bytes=4096)
BIG = 2 ** 32 + 1                                    # a size_t that an int would read as 1


def _call(entry, **bad):
    assert bad, "a call with no bad argument would launch"
    a = {**GOOD, **bad}
    lib = _lib.load()
    head = (a["q"], 0, a["out"], a["Hq"], a["Hkv"], a["D"])
    pages = (a["M"], a["max_seq_len"], a["T"], a["kv"], a["page_list"], a["seq_lens"])
    tail = (a["ws"], a["ws_bytes"], None)
    if entry == "plain":
        rc = lib.b200_paged_decode_attn(*head, a["batch"], *pages, 1.0, *tail)
    elif entry == "multi":
        rc = lib.b200_paged_decode_attn_multi(*head, a["batch"], a["slots"], *pages, 1.0, *tail)
    elif entry == "rope":
        rc = lib.b200_paged_decode_attn_rope(*head, a["batch"], *pages, 1.0, a["rope_base"], *tail)
    elif entry == "beam":
        rc = lib.b200_paged_decode_attn_beam(*head, a["batch"], a["slots"], *pages, a["extra"], 1.0, *tail)
    elif entry == "prefix":
        rc = lib.b200_paged_decode_attn_prefix(*head, a["batch"], a["chunks"], a["slots"], a["offsets"], a["rows"], a["extra"],
                                               *pages, 1.0, *tail)
    else:
        rc = lib.b200_paged_decode_attn_tree(*head, a["batch"], a["slots"], *pages, a["extra"], 1.0, *tail)
    return rc, lib.b200_last_error()


def _r256(n):
    return (n + 255) // 256 * 256


def _workspace_case(entry):
    """Bad arguments that leave the workspace too small for a split merged through L2, and the bytes the message names: a
    counter per (sequence, kv head), then (m, l) and a D-float partial per (query row, split)."""
    bad = dict(M=1024, max_seq_len=65536, ws=None, ws_bytes=0)
    ns = ctypes.c_int()
    tps = ctypes.c_int()
    assert _lib.load().b200_plan_attn_split(GOOD["chunks"] * GOOD["Hkv"], bad["max_seq_len"], ctypes.byref(ns), ctypes.byref(tps)) == 0
    assert ns.value > 8
    seqs, rows = GOOD["batch"], (1 if entry in ("plain", "rope", "prefix") else GOOD["slots"])
    slots = seqs * GOOD["Hq"] * rows * ns.value
    need = _r256(seqs * GOOD["Hkv"] * 4) + _r256(slots * 2 * 4) + slots * GOOD["D"] * 4
    return bad, f"paged_decode_attn: workspace too small (0 < {need})"


def _grid_case(entry):
    unit = {"beam": "requests", "prefix": "chunks"}.get(entry, "batch")
    who = {"beam": "paged_decode_attn_beam", "prefix": "paged_decode_attn_prefix"}.get(entry, "paged_decode_attn")
    return dict(batch=40000, chunks=40000), f"{who}: {unit}*kv_heads 80000 exceeds grid limit"


# checks every entry makes, with the message each gives
COMMON = [
    (dict(out=None), "paged_decode_attn: null pointer"),
    (dict(kv=None), "paged_decode_attn: null pointer"),
    (dict(page_list=None), "paged_decode_attn: null pointer"),
    (dict(seq_lens=None), "paged_decode_attn: null pointer"),
    (dict(D=96), "paged_decode_attn: head_dim 96 unsupported (64 / 128 / 256)"),
    (dict(Hq=6, Hkv=4), "head_num 6 not a multiple of kv_head_num 4"),
    (dict(Hkv=0), "head_num 8 not a multiple of kv_head_num 0"),
    (dict(Hq=0), "paged_decode_attn: group size 0 unsupported (1..64)"),
    (dict(T=24), "paged_decode_attn: page_size 24 unsupported (16/32/64/128)"),
    (dict(max_seq_len=0), "paged_decode_attn: max_seq_len must be >= 1"),
    (dict(max_seq_len=257), "paged_decode_attn: max_seq_len 257 exceeds page table capacity 256"),
    (dict(kv=P + 8), "paged_decode_attn: misaligned pointer"),
    (dict(q=P + 2), "paged_decode_attn: misaligned pointer"),
]


@pytest.mark.parametrize("entry", ENTRIES)
def test_every_entry_makes_the_common_checks(entry):
    gqa = "paged_decode_attn_prefix" if entry == "prefix" else "paged_decode_attn"
    for bad, msg in COMMON + [_workspace_case(entry), _grid_case(entry)]:
        if msg.startswith("head_num"):
            msg = f"{gqa}: {msg}"
        rc, err = _call(entry, **bad)
        assert rc == -1 and msg.encode() in err, (bad, err)


# the checks of one mode that the tests of that mode do not make already
MODE = {
    "plain": [
        (dict(q=None), "paged_decode_attn: null pointer"),
        (dict(Hq=130, Hkv=2), "paged_decode_attn: group size 65 unsupported (1..64)"),
    ],
    "multi": [
        (dict(q=None), "paged_decode_attn_multi: null pointer"),
        (dict(slots=0), "paged_decode_attn_multi: q_len 0 unsupported (1..64)"),
        (dict(slots=BIG), f"paged_decode_attn_multi: q_len {BIG} unsupported (1..64)"),
        (dict(slots=17), "paged_decode_attn: group 4 x q_len 17 exceeds the limit of 64 query rows per (sequence, kv head)"),
    ],
    "rope": [
        (dict(q=None), "paged_decode_attn_rope: null pointer"),
        (dict(rope_base=1.0), "paged_decode_attn_rope: rope_base must be > 1"),
        (dict(rope_base=float("nan")), "paged_decode_attn_rope: rope_base must be > 1"),
        (dict(D=64), "paged_decode_attn_rope: the fused rope is built for head_dim 128 (got 64)"),
        (dict(Hq=34, Hkv=2), "paged_decode_attn_rope: group size 17 unsupported (1..16)"),
    ],
    "beam": [
        (dict(slots=65), "paged_decode_attn_beam: beam_width 65 unsupported (1..64)"),
        (dict(slots=BIG), f"paged_decode_attn_beam: beam_width {BIG} unsupported (1..64)"),
        (dict(extra=None), "paged_decode_attn_beam: null pointer (q or shared_lengths)"),
        (dict(Hq=130, Hkv=2, slots=1), "paged_decode_attn: group size 65 unsupported (1..64)"),
    ],
    "prefix": [
        (dict(q=None), "paged_decode_attn_prefix: null pointer (q or a chunk array)"),
        (dict(offsets=None), "paged_decode_attn_prefix: null pointer (q or a chunk array)"),
        (dict(rows=None), "paged_decode_attn_prefix: null pointer (q or a chunk array)"),
        (dict(extra=None), "paged_decode_attn_prefix: null pointer (q or a chunk array)"),
        (dict(chunks=0), "paged_decode_attn_prefix: chunks 0 must be in 1..batch (2)"),
        (dict(chunks=3), "paged_decode_attn_prefix: chunks 3 must be in 1..batch (2)"),
        (dict(batch=70000), "paged_decode_attn_prefix: batch 70000 exceeds 65535 rows"),
        (dict(slots=0), "paged_decode_attn_prefix: group 4 x max_members 0 exceeds the limit of 64 query rows per (chunk, kv head)"),
        (dict(slots=17), "paged_decode_attn_prefix: group 4 x max_members 17 exceeds the limit of 64 query rows per (chunk, kv head)"),
        (dict(slots=BIG), f"paged_decode_attn_prefix: group 4 x max_members {BIG} exceeds the limit"),
    ],
    "tree": [
        (dict(q=None), "paged_decode_attn_tree: null pointer (q or tree_parents)"),
        (dict(slots=BIG), f"paged_decode_attn_tree: q_len {BIG} unsupported (1..64)"),
        (dict(slots=17), "paged_decode_attn: group 4 x q_len 17 exceeds the limit of 64 query rows per (sequence, kv head)"),
    ],
}


@pytest.mark.parametrize("entry", ENTRIES)
def test_mode_checks(entry):
    for bad, msg in MODE[entry]:
        rc, err = _call(entry, **bad)
        assert rc == -1 and msg.encode() in err, (bad, err)


# An empty call (no sequences, requests or rows) does no work, but some entries check an argument first: the query slots of
# the multi, beam and tree entries and the fused rope's base. Status of each empty call with one otherwise-bad argument.
EMPTY = {
    "plain": [(dict(D=96), 0), (dict(q=None), 0), (dict(out=None), 0), (dict(Hkv=0), 0), (dict(max_seq_len=0), 0)],
    "multi": [(dict(slots=0), -1), (dict(slots=65), -1), (dict(D=96), 0), (dict(q=None), 0), (dict(slots=17), 0)],
    "rope": [(dict(rope_base=1.0), -1), (dict(D=64), 0), (dict(q=None), 0), (dict(Hq=34), 0)],
    "beam": [(dict(slots=0), -1), (dict(slots=65), -1), (dict(extra=None), 0), (dict(D=96), 0), (dict(slots=17), 0)],
    "prefix": [(dict(chunks=0), 0), (dict(chunks=3), 0), (dict(slots=0), 0), (dict(slots=17), 0), (dict(offsets=None), 0),
               (dict(D=96), 0), (dict(Hkv=0), 0)],
    "tree": [(dict(slots=0), -1), (dict(slots=65), -1), (dict(extra=None), 0), (dict(D=96), 0)],
}


@pytest.mark.parametrize("entry", ENTRIES)
def test_empty_calls(entry):
    for bad, status in EMPTY[entry]:
        rc, err = _call(entry, batch=0, **bad)
        assert rc == status, (bad, rc, err)
