"""ctypes binding of libb200_decode.so (include/b200_decode_ops.h). Fails loudly: there is no CPU or PyTorch fallback."""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_size_t, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(HERE, "libb200_decode.so")   # override: developer A/B builds

B200_FMT_F16, B200_FMT_INT8, B200_FMT_INT4, B200_FMT_INT8G = 0, 1, 2, 3
B200_FMT_INT4_G64, B200_FMT_INT4_G32 = 4, 5
B200_GEMM_PDL = 1
B200_GEMM_SILU_MUL = 2

# name -> (restype, argtypes): mirrors include/b200_decode_ops.h one to one (tests check every symbol resolves)
SIGNATURES = {
    "b200_last_error": (c_char_p, []),
    "b200_device_check": (c_int, [c_int]),
    "b200_launch_count": (c_uint64, []),
    "b200_set_pdl": (c_int, [c_int]),
    "b200_plan_attn_split": (c_int, [c_int, c_int, c_void_p, c_void_p]),
    "b200_plan_gemm_split": (c_int, [c_int, c_int, c_void_p, c_void_p]),
    "b200_wo_gemm_max_active_clusters": (c_int, [c_int, c_void_p]),
    "b200_convert_block_table": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "b200_paged_attn_plan": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p] * 5 + [c_void_p]),
    "b200_paged_decode_attn_workspace_bytes": (c_size_t, [c_size_t] * 4),
    "b200_paged_decode_attn": (c_int, [c_void_p, c_int, c_void_p] + [c_size_t] * 7 + [c_void_p, c_void_p, c_void_p,
                                       c_float, c_void_p, c_size_t, c_void_p]),
    "b200_paged_decode_attn_multi": (c_int, [c_void_p, c_int, c_void_p] + [c_size_t] * 8 + [c_void_p, c_void_p, c_void_p,
                                             c_float, c_void_p, c_size_t, c_void_p]),
    "b200_paged_decode_attn_rope": (c_int, [c_void_p, c_int, c_void_p] + [c_size_t] * 7 + [c_void_p, c_void_p, c_void_p,
                                            c_float, c_float, c_void_p, c_size_t, c_void_p]),
    "b200_paged_decode_attn_beam": (c_int, [c_void_p, c_int, c_void_p] + [c_size_t] * 8 + [c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_float, c_void_p, c_size_t, c_void_p]),
    "b200_paged_decode_attn_tree": (c_int, [c_void_p, c_int, c_void_p] + [c_size_t] * 8 + [c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_float, c_void_p, c_size_t, c_void_p]),
    "b200_wo_gemm_packed_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_pack_w4": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_pack_w8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200_pack_w8g": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_wo_gemm_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_wo_gemm": (c_int, [c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_size_t, c_int, c_void_p]),
    "b200_wo_gemm_rs": (c_int, [c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200_add_rmsnorm": (c_int, [c_void_p] * 4 + [c_int, c_int, c_int, c_float, c_void_p]),
    "b200_qk_rmsnorm": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_float, c_void_p]),
    "b200_silu_and_mul": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b200_permute_cols": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b200_rope_append": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_float, c_void_p]),
    "b200_rope_append_multi": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_float, c_int, c_void_p]),
    "b200_rope_append_ex": (c_int, [c_void_p] * 8 + [c_int, c_void_p] + [c_int] * 8 + [c_void_p]),
    "b200_rope_append_ex_multi": (c_int, [c_void_p] * 8 + [c_int, c_void_p] + [c_int] * 9 + [c_void_p]),
    "b200_qk_norm_rope_append": (c_int, [c_void_p] * 3 + [c_float] + [c_void_p] * 4 + [c_int] * 7 + [c_float, c_int, c_void_p]),
    "b200_qk_norm_rope_append_ex": (c_int, [c_void_p] * 3 + [c_float] + [c_void_p] * 6 + [c_int, c_void_p] + [c_int] * 9
                                    + [c_void_p]),
    "b200_embedding": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b200_argmax": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200_sample": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int] + [c_void_p] * 14),
    "b200_spec_verify": (c_int, [c_void_p] * 5 + [c_int] * 3 + [c_void_p] * 3),
    "b200_spec_verify_tree": (c_int, [c_void_p] * 5 + [c_int] * 3 + [c_void_p] * 4),
    "b200_kv_compact_path": (c_int, [c_void_p] + [c_int] * 4 + [c_void_p, c_int] + [c_void_p] * 3 + [c_int, c_int, c_void_p]),
    "b200_beam_search_step_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_beam_search_step": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 4 + [c_void_p] * 7 + [c_size_t, c_void_p]),
    "b200_beam_hypotheses_state_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_beam_hypotheses_update": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p,
                                                                         c_void_p]),
    "b200_beam_hypotheses_finalize": (c_int, [c_void_p, c_size_t] + [c_void_p] * 4 + [c_int] * 6 + [c_void_p] * 6),
    "b200_token_logprobs_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200_token_logprobs": (c_int, [c_void_p] + [c_int] * 4 + [c_void_p] * 5 + [c_size_t, c_void_p]),
    "b200_ban_repeat_ngram": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b200_constrain_logits": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int] + [c_void_p] * 4),
    "b200_peer_ar_region_bytes": (c_size_t, [c_size_t]),
    "b200_peer_alloc": (c_int, [c_size_t, c_void_p, c_void_p]),
    "b200_peer_open": (c_int, [c_void_p, c_void_p]),
    "b200_peer_allreduce": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "b200_peer_allreduce_norm": (c_int, [c_void_p] * 4 + [c_int, c_int, c_int, c_float, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200_peer_gather_norm": (c_int, [c_void_p] * 4 + [c_int, c_int, c_int, c_float, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200_peer_argmax": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200_program_create": (c_int, [c_void_p]),
    "b200_program_begin": (c_int, [c_void_p]),
    "b200_program_end": (c_int, [c_void_p]),
    "b200_program_launch": (c_int, [c_void_p, c_void_p]),
    "b200_program_num_ops": (c_int, [c_void_p]),
    "b200_program_num_launches": (c_int, [c_void_p]),
    "b200_program_set_trace": (c_int, [c_void_p, c_void_p]),
    "b200_program_destroy": (c_int, [c_void_p]),
}



class RopeConfig(ctypes.Structure):
    """b200_rope_config (include/b200_decode_ops.h) = the RopeConfig fields the decode path reads (RopeConfig.h:21-42)."""
    _fields_ = [("style", c_int), ("dim", c_int), ("base", c_float), ("scale", c_float), ("factor1", c_float), ("factor2", c_float),
                ("max_pos", c_int), ("extrapolation_factor", c_float), ("mscale", c_float)]


_lib = None


class B200Error(RuntimeError):
    """Raised for every non-zero status of the C ABI (mirrors RTP_LLM_CHECK_WITH_INFO -> RuntimeError in the reference,
    rtp_llm/cpp/utils/AssertUtils.h:18-27)."""


def _rebuild_if_stale() -> None:
    """The library exists: make sure it was built from the sources next to it (content digest recorded by build.py). A stale
    library is rebuilt under a file lock (several ranks may get here at once); if that is impossible the load fails loudly --
    an edited kernel must never run against an old binary."""
    if os.environ.get("B200_LIB_PATH"):
        return                                    # an explicitly chosen library (developer builds) is taken as it is
    from . import build as _build
    try:
        if _build.stamp_matches():
            return
    except OSError:
        return                                    # sources not shipped with the library: nothing to compare against
    import fcntl
    with open(LIB_PATH + ".lock", "w") as lk:
        fcntl.flock(lk, fcntl.LOCK_EX)
        try:
            if not _build.stamp_matches():        # (another process may have rebuilt it while we waited)
                try:
                    _build.build(force=True)
                except Exception as e:  # noqa: BLE001
                    raise B200Error(f"{LIB_PATH} is older than the sources in {os.path.dirname(LIB_PATH)}/csrc and could not be "
                                    f"rebuilt ({e}): run `python -m rtp_llm_b200.build`") from e
        finally:
            fcntl.flock(lk, fcntl.LOCK_UN)


def load() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            # not a fallback: the only thing we ever do about a missing native library is build the native library
            try:
                from . import build as _build
                _build.build()
            except Exception as e:  # noqa: BLE001
                raise B200Error(f"{LIB_PATH} is missing and could not be built ({e}): run `python -m rtp_llm_b200.build` "
                                "(nvcc, sm_90a). There is no fallback path.") from e
        else:
            _rebuild_if_stale()
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the header and the library ever diverge
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load().b200_last_error().decode()
        raise B200Error(f"{what} failed (status {status}): {msg}")
