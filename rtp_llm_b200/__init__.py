"""rtp_llm_b200 -- Hopper-native (H100, sm_90a) decode hot path of alibaba/rtp-llm: paged decode attention + weight-only
INT4/INT8 x FP16 GEMM behind the reference's op seams. (The directory is `rtp_llm_b200`, not `rtp-llm_b200`: a hyphen is
not importable.)  Compute lives in libb200_decode.so (csrc/, C ABI in include/b200_decode_ops.h); there is no CPU fallback."""
__all__ = ["ops", "build"]
