"""CPU tests of the beam attention's host side: b200_paged_decode_attn_beam rejects bad arguments before any CUDA call, each
with a message that names it, and attention.beam_rows_fit is the rule of when a request's beams share a CTA."""
import ctypes

from rtp_llm_b200 import _lib
from rtp_llm_b200.attention import beam_rows_fit


def _call(Hq=8, Hkv=2, D=128, requests=2, W=4, q=True, shared=True):
    lib = _lib.load()
    buf = (ctypes.c_uint8 * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = lib.b200_paged_decode_attn_beam(p if q else None, 0, p, Hq, Hkv, D, requests, W, 4, 256, 64, p, p, p, p if shared else None,
                                         1.0, p, 4096, None)
    return rc, lib.b200_last_error()


def test_bad_arguments_are_rejected_by_name():
    rc, msg = _call(W=0)
    assert rc == -1 and b"beam_width 0" in msg
    rc, msg = _call(Hq=32, Hkv=8, W=17)                     # group 4 x 17 beams = 68 query rows
    assert rc == -1 and b"group 4 x beam_width 17" in msg and b"64 query rows" in msg
    rc, msg = _call(Hq=64, Hkv=8, W=9)                      # group 8 x 9
    assert rc == -1 and b"group 8 x beam_width 9" in msg
    rc, msg = _call(shared=False)
    assert rc == -1 and b"shared_lengths" in msg
    rc, msg = _call(q=False)
    assert rc == -1 and b"null pointer" in msg
    rc, msg = _call(Hq=32, Hkv=8, requests=8192)            # 8192 x 8 = 65536 CTAs along y
    assert rc == -1 and b"requests*kv_heads 65536 exceeds grid limit" in msg
    rc, msg = _call(D=96)
    assert rc == -1 and b"head_dim 96" in msg


def test_no_requests_is_not_an_error():
    assert _call(requests=0)[0] == 0
    assert _call(requests=0, q=False, shared=False)[0] == 0


def test_beam_rows_fit_is_several_beams_within_64_query_rows_on_at_least_128_pairs():
    assert not beam_rows_fit(32, 8, 1, 32)
    assert beam_rows_fit(32, 8, 2, 32) and beam_rows_fit(32, 8, 16, 16) and not beam_rows_fit(32, 8, 17, 16)
    assert not beam_rows_fit(32, 8, 32, 32)
    assert beam_rows_fit(64, 8, 8, 16) and not beam_rows_fit(64, 8, 16, 16)
    # both sides of the measured boundary: 16 requests x 8 kv heads win, 8 x 8 do not
    assert beam_rows_fit(32, 8, 4, 16) and not beam_rows_fit(32, 8, 4, 8) and not beam_rows_fit(32, 8, 16, 4)
    assert beam_rows_fit(4, 4, 32, 32) and not beam_rows_fit(64, 1, 1, 128)
