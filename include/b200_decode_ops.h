/*
 * b200_decode_ops.h -- C ABI of libb200_decode.so: the Hopper-native (H100, sm_90a) decode hot path of rtp-llm.
 *
 * This is the drop-in boundary.  Every entry point takes plain device pointers, sizes and a cudaStream_t (passed as
 * void*), returns 0 on success or a negative B200_E* code (message via b200_last_error()), never synchronises the
 * stream, never allocates device memory and is CUDA-graph capturable.  No torch types cross this boundary.
 *
 * Each function names the reference interface it replaces (paths relative to the rtp-llm repo root).
 * INTEGRATION.md shows the reference-side binding for each.
 */
#ifndef B200_DECODE_OPS_H
#define B200_DECODE_OPS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_EINVAL (-1)      /* bad argument (shape, alignment, unsupported configuration) */
#define B200_ECUDA (-2)       /* a CUDA runtime / driver call failed */
#define B200_EUNSUPPORTED (-3) /* not an sm_90 device, or feature outside the built scope */

/* weight formats of b200_wo_gemm */
#define B200_FMT_F16 0   /* W stored [N][K] (K contiguous), element type = activation type */
#define B200_FMT_INT8 1  /* per-column symmetric INT8 (device_impl.py:183-222), packed by b200_pack_w8 */
#define B200_FMT_INT4 2  /* GPTQ/AWQ group-128 INT4 (device_impl.py:242-300), packed by b200_pack_w4 */
#define B200_FMT_INT8G 3 /* GPTQ/AWQ group-128 INT8 (device_impl.py:256-258 is_int8 branch: q_s = q_u - 128), packed by b200_pack_w8g */
#define B200_FMT_INT4_G64 4 /* GPTQ/AWQ group-64 INT4, packed by b200_pack_w4 with group 64 */
#define B200_FMT_INT4_G32 5 /* GPTQ/AWQ group-32 INT4, packed by b200_pack_w4 with group 32 */

/* flags of b200_wo_gemm */
#define B200_GEMM_PDL 1  /* launch with programmatic dependent launch (weights prefetched before the upstream grid ends) */
#define B200_GEMM_SILU_MUL 2 /* fused SiLU(gate)*up epilogue: the weight's columns were interleaved per 128-feature tile as
                                [64 gate | 64 matching up] BEFORE packing (rtp_llm_b200.ops.interleave_gate_up); y is [B][N/2] */

/* Last error message of the calling thread ("" if none). */
const char* b200_last_error(void);

/* 0 if device `device` is sm_90 (H100) and the library's kernels can run there, else B200_EUNSUPPORTED. */
int b200_device_check(int device);

/* Library-wide switch: launch the kernels of the decode chain (norms, rope, attention, GEMMs) with programmatic dependent
 * launch so each kernel's launch latency / prologue / weight prefetch overlaps its predecessor's tail. Every such kernel
 * executes griddepcontrol.wait before touching dependent data, so results are unchanged. Default off. */
int b200_set_pdl(int enable);

/* Number of kernels this library has launched since load (all threads); used by bench.py for "gpu_launches". */
uint64_t b200_launch_count(void);

/* Launch shapes the library will choose (host-only, no CUDA work): how many sequence splits / 64-token tiles per CTA the
 * attention takes for `units` = batch*kv_heads and a given max_seq_len, and the split-K of a GEMM. For capacity planning
 * (workspaces) and for tests of the heuristics. */
int b200_plan_attn_split(int units, int max_seq_len, int* nsplit, int* tiles_per_split);
int b200_plan_gemm_split(int K, int N, int* nsplit, int* k_blocks_per_split);
/* Diagnostic: thread-block clusters of cluster_size (1..8) CTAs of the weight-only GEMM kernel (INT4 group 128, FP16, batch
 * pad 32) that the current device holds co-resident (cudaOccupancyMaxActiveClusters). */
int b200_wo_gemm_max_active_clusters(int cluster_size, int* num_clusters);

/* ------------------------------------------------------------------------------------------------ indexing */

/* Replaces invokeConvertOffsetToBlockArrayData
 *   rtp_llm/models_py/bindings/common/kernels/kv_cache_kernels.cu:66-80 (kernel :49-63).
 * block_ids [batch][max_blocks] int32 -> page_list [batch][1][2][max_blocks] int32, K page = 2*id, V page = 2*id+1. */
int b200_convert_block_table(int32_t* page_list, const int32_t* block_ids, int batch, int max_blocks, void* stream);

/* Replaces invokeMhaPagedAttnPlan  rtp_llm/models_py/bindings/cuda/kernels/mha_paged_attn_plan.cu:100-180 (kernel :16-97).
 * prefix_lengths == NULL selects decode mode (one token per sequence, seq_len = sequence_lengths[b]+1).
 * block_ids may be NULL (page_indice untouched). batch <= 1024. */
int b200_paged_attn_plan(const int32_t* input_lengths, const int32_t* sequence_lengths, const int32_t* prefix_lengths,
                         const int32_t* block_ids, int batch, int max_blocks, int tokens_per_block,
                         int32_t* paged_kv_last_page_len, int32_t* decode_page_indptr, int32_t* page_indice,
                         int32_t* batch_indice, int32_t* positions, void* stream);

/* ------------------------------------------------------------------------------------------------ attention */

/* Bytes of scratch b200_paged_decode_attn needs for this problem size. The buffer must be zero-filled ONCE after
 * allocation (cudaMemset); the kernels leave it zeroed where it matters (semaphores self-reset). */
size_t b200_paged_decode_attn_workspace_bytes(size_t batch, size_t head_num, size_t kv_head_num, size_t max_seq_len);

/* Replaces runXqa  rtp_llm/models_py/bindings/cuda/ops/CudaXqa.h:65-84 (called from XQAAttnOp::forward,
 * rtp_llm/models_py/bindings/cuda/XQAAttnOp.cc:119-156) and the flashinfer trtllm-gen call at
 * rtp_llm/models_py/modules/factory/attention/cuda_impl/trtllm_gen.py:531-545.
 *   q            [batch][head_num][head_dim]                        fp16 / bf16
 *   out          [batch][head_num*head_dim]                         same type
 *   kv_pool      layer cache [pages][2][kv_head_num][page_size][head_dim] (OpDefs.h:201-202), addressed as a pool of
 *                2*pages pages of [kv_head_num][page_size][head_dim]
 *   page_list    [batch][1][2][max_blocks_per_seq] int32 from b200_convert_block_table
 *   sequence_lengths [batch] tokens ALREADY in the cache (device-accessible; pinned host memory works, as in the
 *                reference); attention covers positions 0..sequence_lengths[b] inclusive
 *   max_seq_len  host upper bound of sequence_lengths[b]+1 (sizes the sequence split; as XQAAttnOp.cc:149)
 *   softmax scale = q_scale * head_dim^-1/2.
 * Supported: head_dim 64 / 128 / 256, head_num/kv_head_num in 1..64, page_size in {16,32,64,128}. */
int b200_paged_decode_attn(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                           size_t batch, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                           const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                           float q_scale, void* workspace, size_t workspace_bytes, void* stream);

/* q_len > 1 query tokens per sequence (verification of speculative tokens: runXqa's max_q_len, CudaXqa.h:59-84; trtllm-gen's
 * q_len_per_req, trtllm_gen.py:544): q [batch][q_len][head_num][head_dim], out [batch][q_len][head_num*head_dim]; the K/V of all
 * q_len new tokens are already in the cache; sequence_lengths[b] = tokens cached BEFORE them, query j attends to positions
 * 0 .. sequence_lengths[b] + j. (head_num / kv_head_num) * q_len <= 64; max_seq_len bounds sequence_lengths[b] + q_len; size the
 * workspace with b200_paged_decode_attn_workspace_bytes(batch * q_len, ...). q_len == 1 is b200_paged_decode_attn. */
int b200_paged_decode_attn_multi(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                 size_t batch, size_t q_len, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                 const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths, float q_scale,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* The same attention with RoPE + KV append FUSED IN (what XQA does with USE_INPUT_KV + ROPE_STYLE, 3rdparty/xqa/mha.h:82-86):
 * replaces FusedRopeKVCacheDecodeOp.forward + XQAAttnOp.forward (rtp_llm/ops/fused_rope_kvcache_op.py:202-246 then
 * bindings/cuda/XQAAttnOp.cc:119-156) by one launch. `qkv` is the qkv GEMM output [batch][(head_num + 2 kv_head_num) * head_dim],
 * un-rotated; q is rotated on load, the CTA that owns the tile of position sequence_lengths[b] rotates k and appends k, v to
 * `kv_pool` before streaming it. RopeStyle::Base, NeoX pairing, same arithmetic as b200_rope_append: cache contents and attention
 * output are bit-identical to the two-call sequence. head_num / kv_head_num <= 16 (one token per sequence). */
int b200_paged_decode_attn_rope(const void* qkv, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t batch, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size, void* kv_pool,
                                const int32_t* page_list, const uint32_t* sequence_lengths, float q_scale, float rope_base,
                                void* workspace, size_t workspace_bytes, void* stream);

/* Beam search: the attention of `requests` requests with beam_width beams each, reading what a request's beams share once for all
 * of them. Replaces runXqa with XQAParams::beam_width > 1 (CudaXqa.h:10-16, 65-84; XQA's beamWidth, 3rdparty/xqa/mha_sm90.cu:
 * ctaNbValidQHeads = headGrpSize * beamWidth), which b200_paged_decode_attn serves as requests * beam_width unrelated sequences.
 *   q, out, page_list, sequence_lengths   those of b200_paged_decode_attn with batch = requests * beam_width; row
 *                b * beam_width + i is beam i of request b. Beams of a request may differ in length.
 *   shared_lengths [requests] int32 (device-accessible): tokens of each request that all its beams share. Over the first
 *                shared_lengths[b] / page_size pages the request's beam_width page_list rows must be equal; beam 0's are read.
 *                The kernel rounds the value down to a multiple of 64 and keeps it at or below the shortest beam's
 *                sequence_lengths (the token a step appends is never shared), so any value is safe under that contract and
 *                0 shares nothing.
 * Every output row has the bits it has with shared_lengths = 0, whatever is shared, and beam_width == 1 gives the bits of
 * b200_paged_decode_attn. (head_num / kv_head_num) * beam_width <= 64; requests * kv_head_num <= 65535; max_seq_len bounds
 * sequence_lengths[.] + 1; size the workspace with b200_paged_decode_attn_workspace_bytes(requests * beam_width, ...). */
int b200_paged_decode_attn_beam(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t requests, size_t beam_width, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                                const int32_t* shared_lengths, float q_scale, void* workspace, size_t workspace_bytes, void* stream);

/* Verification of a speculative token TREE (EAGLE / Medusa drafts; TensorRT-LLM XQA's spec-decoding mask, restated: parity
 * unpinned). The arguments of b200_paged_decode_attn_multi plus tree_parents [batch][q_len] int32 (device): the q_len new tokens of
 * sequence b are nodes, node 0 the root (the last accepted token; its entry is not read), node j >= 1 under tree_parents[b][j] in
 * [0, j). Node j's K/V sit at slot sequence_lengths[b] + j. Query j attends to positions 0 .. sequence_lengths[b] - 1 and to the
 * slots of the nodes on its ancestor walk: j, its parent, ... up to the root or to a parent outside [0, i), which ends the walk.
 * No value of tree_parents reads outside its row. A chain (parents[j] = j - 1) gives the bits of b200_paged_decode_attn_multi.
 * A new token outside a query's ancestors never changes that query's bits, even when its K/V hold NaN or inf: its non-finite V
 * elements are read as 0, and a query whose ancestors hold one gets a NaN output row. Same limits and workspace sizing as
 * b200_paged_decode_attn_multi. */
int b200_paged_decode_attn_tree(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t batch, size_t q_len, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                                const int32_t* tree_parents, float q_scale, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------ weight-only GEMM */

/* Load-time weight re-layout.  Replace CudaImpl.preprocess_weights_for_mixed_gemm (rtp_llm/device/device_impl.py:392-479):
 * instead of the FT sm80 interleave, weights become per-(128 features x 128 k) blobs that one TMA bulk copy stages.
 * Inputs are the loader's UN-permuted tensors (device pointers):
 *   b200_pack_w4: q_packed uint8 [K][N/2] (low nibble = even column, two's complement q_s = q_u - 8, device_impl.py:204-209),
 *                 scales, zeros_x_scales [K/group][N] 16-bit in the ACTIVATION type (fp16 or bf16); group 128, 64 or 32
 *                 selects the blob format B200_FMT_INT4 / _INT4_G64 / _INT4_G32. Blob per block: 8192 bytes of nibbles, then
 *                 group 128: 128 scales and 128 zeros_x_scales; group 64 / 32: per group in k order, 128 {scale, zeros_x_scale}
 *                 pairs (9216 / 10240 bytes per block)
 *   b200_pack_w8: q int8 [K][N] (device_impl.py:183-202); the per-column scale stays a separate [N] tensor
 *   b200_pack_w8g: q int8 [K][N] (8-bit group-wise checkpoints, q_s = q_u - 128, device_impl.py:256-274) + scales,
 *                 zeros_x_scales [K/128][N] as for b200_pack_w4; dequant W' = q_s * s + zeros_x_scales (device_impl.py:284-291)
 * K % 128 == 0; N % 2 == 0 (int4). Output size: b200_wo_gemm_packed_bytes(fmt, K, N). */
size_t b200_wo_gemm_packed_bytes(int fmt, int K, int N);
int b200_pack_w4(const uint8_t* q_packed, const void* scales, const void* zeros_x_scales, int K, int N, int group,
                 void* blob, void* stream);
int b200_pack_w8(const int8_t* q, int K, int N, void* blob, void* stream);
int b200_pack_w8g(const int8_t* q, const void* scales, const void* zeros_x_scales, int K, int N, int group, void* blob,
                  void* stream);

/* Scratch for split-K / stream-K partials + semaphores (+ the grid-barrier words of a stand-alone call); zero-fill once
 * after allocation (the kernels leave the semaphores at zero). Required for INT8 / INT4 weights, and for any weight format
 * whose split-K plan splits K (at least 24 KiB); b200_wo_gemm rejects a smaller one. */
size_t b200_wo_gemm_workspace_bytes(int max_batch, int N, int K);

/* Y[B][N] = X[B][K] . W' (+ bias).  The compute behind LinearBase.forward
 * (rtp_llm/models_py/modules/factory/linear/linear_base.py:81; call sites modules/hybrid/causal_attention.py:83,90,
 * dense_mlp.py:99,103; lm_head cpp/models/PyWrappedModel.cc:1041-1046) for weight-only INT4/INT8 and FP16 weights.
 *   w         B200_FMT_INT4/INT4_G64/INT4_G32/INT8/INT8G: blob from b200_pack_w4/8/8g; B200_FMT_F16: W [N][K] (K contiguous)
 *   col_scale INT8 only: [N] per-column scale in the activation type
 *   bias      optional [N]
 * B <= 128, K % 128 == 0, x / y / w 16-byte aligned. */
int b200_wo_gemm(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* col_scale,
                 const void* bias, void* y, void* workspace, size_t workspace_bytes, int flags, void* stream);

/* ------------------------------------------------------------------------------------------------ glue ops (SURVEY 8f) */

/* fused_add_rmsnorm / rmsnorm (rtp_llm/models_py/bindings/cuda/RegisterBaseBindings.hpp:45-160).
 * residual may be NULL; otherwise residual += x (in place) and y = rmsnorm(residual) * gamma. hidden % 8 == 0. */
int b200_add_rmsnorm(const void* x, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                     float eps, void* stream);
/* Per-head RMSNorm of the q and k heads of qkv [rows][(head_num + 2 kv_head_num) * head_dim], in place (QK-norm before RoPE):
 * invokeFusedQkRmsNorm, rtp_llm/models_py/bindings/cuda/kernels/fused_qk_rmsnorm.cu:80-150 (call site model_desc/qwen3.py:57-79).
 * gamma / bias are [head_dim]; biases optional (both or none); head_dim % 64 == 0. */
int b200_qk_rmsnorm(void* qkv, const void* q_gamma, const void* k_gamma, const void* q_bias, const void* k_bias, int is_bf16,
                    int rows, int head_num, int kv_head_num, int head_dim, float eps, void* stream);
/* silu_and_mul: y[r][c] = silu(gate_up[r][c]) * gate_up[r][inter + c]. */
int b200_silu_and_mul(const void* gate_up, void* y, int is_bf16, int rows, int inter, void* stream);
/* Column gather y[r][j] = x[r][perm[j]] over x, y [rows][K] fp16 / bf16 (a bit copy): the input of a GEMM whose weight is a GPTQ
 * act-order (desc_act) weight with its rows sorted by g_idx. perm int32 [K] is a permutation of 0..K-1 (not checked here: it
 * is checked once when the weight is packed). x != y; K % 8 == 0, K <= 65536; x, perm, y 16-byte aligned. Inside a decode
 * program it is its own launch. */
int b200_permute_cols(const void* x, const int32_t* perm, void* y, int is_bf16, int rows, int K, void* stream);
/* FusedRopeKVCacheDecodeOp.forward (rtp_llm/ops/fused_rope_kvcache_op.py:202-246), RopeStyle::Base, NeoX pairing:
 * rotates q and k of qkv [B][(Hq+2Hkv)*D] at position sequence_lengths[b], writes q to q_out [B][Hq*D] and K,V of the
 * new token into the paged cache. */
int b200_rope_append(const void* qkv, void* q_out, void* kv_pool, const int32_t* page_list,
                     const int32_t* sequence_lengths, int is_bf16, int batch, int head_num, int kv_head_num,
                     int head_dim, int max_blocks_per_seq, int page_size, float rope_base, void* stream);
/* b200_rope_append for q_len new tokens per sequence (verification of speculative tokens): row x of qkv [batch*q_len][...]
 * is token j = x % q_len of sequence b = x / q_len, rotated and appended at position (and cache slot) sequence_lengths[b] + j;
 * q_out [batch*q_len][Hq*D] is the q [batch][q_len][Hq][D] of b200_paged_decode_attn_multi. q_len == 1 is b200_rope_append.
 * Inside a decode program it is its own launch. */
int b200_rope_append_multi(const void* qkv, void* q_out, void* kv_pool, const int32_t* page_list,
                           const int32_t* sequence_lengths, int is_bf16, int batch, int head_num, int kv_head_num,
                           int head_dim, int max_blocks_per_seq, int page_size, float rope_base, int q_len, void* stream);
/* The full decode contract of FusedRopeKVCacheDecodeOp.forward (rtp_llm/ops/fused_rope_kvcache_op.py:202-246; device code
 * rtp_llm/models_py/bindings/common/kernels/rotary_position_embedding.h:322-442,889-1062). b200_rope_config mirrors the
 * fields of RopeConfig (rtp_llm/cpp/model_utils/RopeConfig.h:21-42) the decode path reads.
 *   position_ids     optional [batch]; an entry > 0 replaces sequence_lengths[b] as the rotation position (:1040-1042);
 *                    K/V are still appended at slot sequence_lengths[b]
 *   cos_sin_cache    optional float2 [cache_positions][dim/2] = (cos, sin), the layout getRopeCache produces with
 *                    interleave = true (cpp/model_utils/RopeCache.cc:16-85; used for Base and Yarn); without it the
 *                    coefficients are computed in the kernel with the reference's formulas
 *   styles           0 No, 1 Base (linear scale), 3 DynamicNTK, 4 QwenDynamicNTK, 5 Yarn, 6 Llama3, 7 Mrope (as Base);
 *                    factor1 / factor2 = beta_slow / beta_fast (Yarn) or low / high frequency factor (Llama3); max_pos =
 *                    original_max_position_embeddings
 *   qkv_bias         optional [(head_num + 2 kv_head_num) * head_dim], added before the rotation
 *   use_logn_attn    q *= log(pos + 1) / log(max_pos) for pos > max_pos
 * NeoX pairing (i, i + dim/2) within the first `dim` channels of a head; the rest pass through. */
typedef struct b200_rope_config {
    int style;
    int dim;
    float base, scale, factor1, factor2;
    int max_pos;
    float extrapolation_factor, mscale;
} b200_rope_config;
int b200_rope_append_ex(const void* qkv, const void* qkv_bias, void* q_out, void* kv_pool, const int32_t* page_list,
                        const int32_t* sequence_lengths, const int32_t* position_ids, const float* cos_sin_cache,
                        int cache_positions, const b200_rope_config* cfg, int use_logn_attn, int is_bf16, int batch, int head_num,
                        int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, void* stream);
/* b200_rope_append_ex for q_len new tokens per sequence (verification of speculative tokens), with the same per-row rules:
 * row x of qkv [batch*q_len][...] is token j = x % q_len of sequence b = x / q_len; its K/V go to slot sequence_lengths[b] + j,
 * and it is rotated at position_ids[x] (position_ids [batch*q_len]) when that entry is > 0, else at that slot. Dynamic-NTK
 * seq_len, the logn factor and the cos_sin_cache bound are taken per row from that position, so token j has the bits of a
 * one-token b200_rope_append_ex at sequence_lengths + j. q_out [batch*q_len][Hq*D] is the q [batch][q_len][Hq][D] of
 * b200_paged_decode_attn_multi. q_len == 1 is b200_rope_append_ex. Inside a decode program it is its own launch. */
int b200_rope_append_ex_multi(const void* qkv, const void* qkv_bias, void* q_out, void* kv_pool, const int32_t* page_list,
                              const int32_t* sequence_lengths, const int32_t* position_ids, const float* cos_sin_cache,
                              int cache_positions, const b200_rope_config* cfg, int use_logn_attn, int is_bf16, int batch,
                              int head_num, int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, int q_len,
                              void* stream);
/* QK-RMSNorm (Qwen3's q_norm / k_norm) + RoPE + K/V append in one launch: b200_rope_append_multi / b200_rope_append_ex_multi
 * after each q and k head of qkv is RMS-normalised with q_gamma / k_gamma [head_dim] and eps. q_out and the K/V pool get the
 * bits of b200_qk_rmsnorm(copy of qkv, q_gamma, k_gamma, NULL, NULL, ..., eps) followed by the rope entry on that copy; v
 * heads are copied as they are and qkv is only read. q_len >= 1 tokens per sequence (1: the one-token entries' rules).
 * head_dim % 64 == 0 and <= 256; both gammas required; no qkv bias (it belongs to the qkv GEMM, before the norm). Inside a
 * decode program each is its own launch (the persistent kernel's rope op does not normalise). */
int b200_qk_norm_rope_append(const void* qkv, const void* q_gamma, const void* k_gamma, float eps, void* q_out, void* kv_pool,
                             const int32_t* page_list, const int32_t* sequence_lengths, int is_bf16, int batch, int head_num,
                             int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, float rope_base, int q_len,
                             void* stream);
int b200_qk_norm_rope_append_ex(const void* qkv, const void* q_gamma, const void* k_gamma, float eps, void* q_out, void* kv_pool,
                                const int32_t* page_list, const int32_t* sequence_lengths, const int32_t* position_ids,
                                const float* cos_sin_cache, int cache_positions, const b200_rope_config* cfg, int use_logn_attn,
                                int is_bf16, int batch, int head_num, int kv_head_num, int head_dim, int max_blocks_per_seq,
                                int page_size, int q_len, void* stream);
/* embedding gather out[b] = table[ids[b]] (rtp_ops.embedding). */
int b200_embedding(const int32_t* ids, const void* table, void* out, int is_bf16, int rows, int hidden, void* stream);
/* greedy sampling: out[r] = argmax(logits[r]) (lowest index on ties; CudaSampleOp.cc:330,453). dtype: 0 fp16, 1 bf16, 2 fp32 */
int b200_argmax(const void* logits, int dtype, int rows, int vocab, int32_t* out, void* stream);

/* Token sampling: the CUDA path behind sampleGreedy (rtp_llm/models_py/bindings/core/CudaSampleOp.cc:423-463; processLogits
 * :186-279, flashinferSampleGreedy :287-421; penalty kernels common/kernels/sampling_penalty_kernels.cu:26-53,129-185).
 * Per row, in this order: temperature (logit *= 1/(T+1e-6)), repetition / presence / frequency penalties over the DISTINCT
 * tokens of `history` (hist_len[r] valid ids of [rows][hist_stride]), softmax (the probabilities REPLACE the logits, as in the
 * reference), top-k (keep p >= the k-th largest; top_k <= 0 = no limit; top_k == 1 = argmax, lowest index on ties), top-p
 * within what is left (smallest set of largest p reaching top_p; |top_p| < 1e-7 or >= 1 = no limit), min-p within what is left
 * (keep p >= fl32(min_p[r] * p_max), p_max the row's largest p; min_p optional [rows], clamped to [0, 1]; NULL or 0 = no limit,
 * bit-identical to a call without it), renormalise, and one inverse-CDF draw in index order with the caller's uniform[r] in [0, 1), which always returns a kept token with p > 0
 * (token -1 and token_prob 0 only for a row without positive finite mass, i.e. NaN logits).  Same distribution as the
 * reference's flashinfer rejection sampler, different random stream: the caller owns the randomness, so the op is
 * deterministic and graph-replayable.
 * process[r] == 0 (do_sample false) skips temperature / penalties for that row. count_ws: [rows][vocab] int32, zero on entry
 * and on exit (only read with penalties). Optional outputs: token_prob_out[r] (renormalised probability of the drawn token,
 * for cum_log_probs += log p), probs_out [rows][vocab] (output_all_probs after renormalisation). logits fp32, contiguous. */
int b200_sample(float* logits, int rows, int vocab, const int32_t* history, const int32_t* hist_len, int hist_stride,
                int32_t* count_ws, const float* temperature, const float* repetition, const float* presence,
                const float* frequency, const int32_t* top_k, const float* top_p, const float* min_p, const float* uniform,
                const uint8_t* process, int32_t* token_out, float* token_prob_out, float* probs_out, void* stream);

/* Verification of num_draft = n speculative tokens per sequence (the chain form of the reference's speculative-sampling kernel,
 * rtp_llm/models_py/bindings/cuda/kernels/speculative_sampling/sampling.cu), after a step over the batch*(n+1) rows
 * [last accepted token, draft 0 .. draft n-1] of each sequence.
 *   draft_tokens [batch][n]; out_tokens [batch][n+1]: the accepted drafts, one correction or bonus token, then -1;
 *   accepted [batch] in 0..n (the sequence advances by accepted + 1).
 * Greedy (target_probs == NULL): target_ids [batch][n+1] (b200_argmax of the rows); accepted = the first i with
 *   draft[i] != target_ids[i] (n if none), the emitted token is target_ids[accepted].
 * Sampling: target_probs [batch][n+1][vocab] fp32 (probs_out of b200_sample over the rows), draft_probs [batch][n][vocab] or
 *   NULL (deterministic drafts, one-hot), uniform [batch][n+1] in [0, 1). Draft i = d is accepted iff uniform[i] * p(d) < q(d)
 *   in fp32 (p = draft_probs[i][d], or 1); at the first rejection the token is drawn from max(0, q - p) (from q when that has
 *   no mass), after n acceptances from target row n, both with uniform[n] by inverse CDF in index order as b200_sample draws
 *   (always a token with positive mass; -1 only for a row without any). Same distribution as the reference, caller-owned
 *   randomness. One CTA per sequence. */
int b200_spec_verify(const float* target_probs, const int32_t* target_ids, const float* draft_probs, const int32_t* draft_tokens,
                     const float* uniform, int batch, int num_draft, int vocab, int32_t* out_tokens, int32_t* accepted, void* stream);

/* Verification of a speculative token tree of n <= 64 nodes per sequence (the tree of b200_paged_decode_attn_tree), after a step
 * over its batch*n rows; b200_spec_verify is the case of a chain, and the two share one kernel.
 *   tree_parents [batch][n] (node 0 the root, node c >= 1 under parents[c] in [0, c); a child with a parent outside that range
 *   is never reached), node_tokens [batch][n] (node c's draft token; entry 0 is not read), uniform [batch][n].
 * The walk starts at the root and tries the current node's children in index order.
 * Greedy (target_probs == NULL): move to the first child whose token equals target_ids[cur]; at none, emit target_ids[cur].
 * Sampling (deterministic drafts, multi-round rejection after SpecInfer / EAGLE): with t = target_probs[cur], child c with token x
 *   is accepted iff uniform[c - 1] * (1 - S) < r(x) in fp32, where r is t with the tokens of the siblings rejected before c
 *   zeroed (a duplicate sibling token has mass 0) and S is the fp32 sum of r over those rejections. With every child rejected the
 *   token is drawn from max(0, t - 1) on the rejected tokens and t elsewhere (from t when that has no mass); at a leaf the bonus
 *   token is drawn from t; both with uniform[n - 1] as b200_spec_verify draws.
 * Outputs: out_tokens [batch][n] the path's tokens at depths 1..a, then the correction or bonus token, then -1; accepted [batch]
 * = a; accepted_path [batch][n] the node at depths 0..a (path[0] = 0), then -1. On a chain every output equals b200_spec_verify's
 * (with out_tokens of n = num_draft + 1 entries). */
int b200_spec_verify_tree(const float* target_probs, const int32_t* target_ids, const int32_t* tree_parents, const int32_t* node_tokens,
                          const float* uniform, int batch, int n, int vocab, int32_t* out_tokens, int32_t* accepted,
                          int32_t* accepted_path, void* stream);

/* After b200_spec_verify_tree: the accepted path's K/V moved to consecutive cache slots. For d = 1 .. accepted[b] with
 * path[d] != d (path = accepted_path [batch][n]), the K and V of slot sequence_lengths[b] + path[d] are bit-copied to slot
 * sequence_lengths[b] + d in every layer and kv head; no other slot is written. Copies go in increasing d, each read before any
 * later write (path [0, 2, 3] reads slot 2 before writing it). kv_pools: a HOST array of `layers` <= 128 per-layer pools
 * [pages][kv_head_num][page_size][head_dim] of 16-bit elements, copied at the call; page_list [batch][2][max_blocks_per_seq] as
 * for attention; sequence_lengths [batch] tokens cached before the step's nodes. accepted is clamped to [0, n - 1], and a path
 * entry outside [0, n) or a slot past the page table is skipped. One launch for all layers; under PDL it waits before reading. */
int b200_kv_compact_path(void* const* kv_pools, int layers, int kv_head_num, int head_dim, int page_size, const int32_t* page_list,
                         int max_blocks_per_seq, const int32_t* sequence_lengths, const int32_t* accepted_path, const int32_t* accepted,
                         int batch, int n, void* stream);

/* One beam-search step over the lm_head logits of `batch` requests x W = beam_width beams. The semantics are restated from the
 * Hugging Face / TensorRT-LLM beam-search convention; the reference's vendored kernels (3rdparty/trt_beam_search) are not in
 * this tree, so parity with them is unpinned, as for the GEMM.
 *   logits [batch*W][vocab] (row b*W + i = beam i of request b), dtype 0 fp16, 1 bf16, 2 fp32, read as they are (no cast);
 *   cum_log_probs fp32 [batch][W]. W in 1..32, vocab >= 2W, ceil(vocab / 4096) * 2W <= 4096, vocab <= 2^26.
 * Every candidate (i, v) scores cum[b][i] + (x - m_i) - log sum_v exp(x - m_i) in fp32 (x the logit, m_i the row max: a log-softmax
 * per beam); candidates rank by score descending, equal scores by lower flat index i*vocab + v. -inf logits and rows with
 * cum = -inf give -inf scores, which rank last, by index (first step: cum[b][1:] = -inf, so only beam 0 contributes).
 * Outputs: the top 2W candidates in rank order, cand_token / cand_parent (beam index 0..W-1) / cand_score [batch][2W]; the next
 * beams next_token / next_parent / next_cum [batch][W] = the first W ranked candidates whose token is not eos_id (-1: none). Each
 * row adds at most one EOS candidate, so W of the 2W are never EOS; the EOS candidates among the first W ranks are the finished
 * hypotheses, which b200_beam_hypotheses_update keeps on the device.
 * workspace: b200_beam_search_step_workspace_bytes(batch, W, vocab) bytes, ZERO on first use; every call leaves it zero-ready
 * (self-resetting arrival counters). One launch, deterministic, graph-capturable; under PDL it waits before reading logits / cum. */
size_t b200_beam_search_step_workspace_bytes(int batch, int beam_width, int vocab);
int b200_beam_search_step(const void* logits, int dtype, const float* cum_log_probs, int batch, int beam_width, int vocab, int eos_id,
                          int32_t* cand_token, int32_t* cand_parent, float* cand_score, int32_t* next_token, int32_t* next_parent,
                          float* next_cum, void* workspace, size_t workspace_bytes, void* stream);

/* The finished-hypothesis set of beam search, per request, on the device (Hugging Face BeamHypotheses / BeamSearchScorer and
 * TRT-LLM's device-side finished candidates, restated; parity with the reference's kernels unpinned). W = beam_width in 1..32.
 * State: b200_beam_hypotheses_state_bytes(batch, W, max_len) bytes owned by the caller; request b owns the stride
 * = 16 + 16*W + 4*W*max_len bytes at b * stride:
 *   int32 count (filled slots, 0..W), int32 next_order (insertion order of the next hypothesis), int32 pad[2];
 *   W slots of {float cum (raw log-prob), float score, int32 len (generated tokens), int32 order}; slots 0..count-1 are filled;
 *   int32 tokens [W][max_len]: slot k's path, its first min(len, max_len) entries (the rest is undefined).
 * All-zero bytes are the empty set, so restarting from the prompt is a memset. done int32 [batch], also caller-owned and zeroed
 * with the state: set once a request is done and never cleared.
 * A hypothesis of raw log-prob cum and L generated tokens scores s = cum / L^alpha in fp32 (exactly cum at alpha 0), alpha =
 * length_penalty[b]. It enters a set of fewer than W, or a full set when s > the set's lowest score (strictly), evicting the
 * lowest (the earliest inserted among equal lowest scores).
 * history [batch*W][hist_stride], hist_len [batch*W] (clamped to hist_stride): each beam's token history; its generated tokens
 * are history[row][gen_start : hist_len[row]] (none when hist_len <= gen_start).
 *
 * b200_beam_hypotheses_update: after b200_beam_search_step (its cand_token / cand_parent / cand_score [batch][2W]) and before
 * the history rows are forked. One CTA per request; a request with done[b] set is skipped entirely. Ranks r = 0..W-1 in order:
 * a candidate whose token is eos_id and whose score is finite becomes a hypothesis with cum = its score, the path of row
 * b*W + cand_parent followed by eos_id (kept up to max_len tokens) and L = that row's generated tokens + 1. EOS at rank >= W is
 * ignored. Then, with a full set, the request is done when early_stopping[b] is 1, or (0, and 2 at alpha <= 0) when
 * worst >= cand_score[b][0] / L^alpha, L the generated length of rank 0's candidate (its parent row's + 1), or (2 = "never",
 * alpha > 0) when worst >= cand_score[b][0] / max_len^alpha. Any other early_stopping value counts as 0. eos_id >= 0.
 * b200_beam_hypotheses_finalize: the n (1..W) best of each request's set into out_tokens [batch][n][max_len], out_len,
 * out_score (= s), out_cum [batch][n], sorted by score descending, the earlier inserted first among equal scores. For a request
 * that is not done, the W live beams are merged in first by the same rule, in rank order: beam i has cum beam_cum[b][i]
 * ([batch][W]) and the path history[b*W + i][gen_start : hist_len] without EOS (a beam with a non-finite cum or no generated
 * token is left out). Token slots past a path are -1; a missing hypothesis has tokens -1, len -1, score and cum -inf. The state
 * and done are only read, so it may run after any step and again later.
 * Both: deterministic, graph-capturable, allocate nothing; under PDL they wait before reading anything. */
size_t b200_beam_hypotheses_state_bytes(int batch, int beam_width, int max_len);
int b200_beam_hypotheses_update(const int32_t* cand_token, const int32_t* cand_parent, const float* cand_score, const int32_t* history,
                                const int32_t* hist_len, int hist_stride, int gen_start, int batch, int beam_width, int eos_id,
                                const float* length_penalty, const int32_t* early_stopping, int max_len, void* state,
                                size_t state_bytes, int32_t* done, void* stream);
int b200_beam_hypotheses_finalize(const void* state, size_t state_bytes, const int32_t* done, const float* beam_cum,
                                  const int32_t* history, const int32_t* hist_len, int hist_stride, int gen_start, int batch,
                                  int beam_width, int n, int max_len, const float* length_penalty, int32_t* out_tokens,
                                  int32_t* out_len, float* out_score, float* out_cum, void* stream);

/* Per-token log-probabilities of the lm_head output (OpenAI-style logprobs / top_logprobs), without copying the probabilities
 * to the host. logits [rows][vocab], dtype 0 fp16, 1 bf16, 2 fp32, read as they are. Each row's lp(i) = (x_i - m) - log sum_v
 * exp(x_v - m) in fp32, m the row max: the log-softmax of the logits AS GIVEN, i.e. the raw model distribution before
 * temperature, penalties and top-k / top-p (what b200_sample draws from is the filtered distribution; its token_prob_out is
 * that one's renormalised probability). NaN logits count as -inf.
 *   token_logprob [rows] = lp(tokens[r]) when tokens [rows] is given (NaN for an id outside [0, vocab));
 *   top_ids int32 / top_logprobs fp32 [rows][top_n]: the top_n largest lp in descending order, equal values by lower id.
 * top_n in 0..64 and <= vocab, with ceil(vocab / 4096) * top_n <= 4096 (at vocab 152064: top_n <= 64); vocab <= 2^26; rows <= 65535.
 * A row without a finite logit gives NaN. Same grid and code as the first two levels of b200_beam_search_step: one CTA per
 * 4096-logit chunk, the last one of a row to arrive merges the row's chunks in a fixed order. workspace:
 * b200_token_logprobs_workspace_bytes(rows, vocab, top_n) bytes, ZERO on first use, left zero-ready by every call. One launch,
 * deterministic, graph-capturable; under PDL it waits before reading anything. */
size_t b200_token_logprobs_workspace_bytes(int rows, int vocab, int top_n);
int b200_token_logprobs(const void* logits, int dtype, int rows, int vocab, int top_n, const int32_t* tokens, float* token_logprob,
                        int32_t* top_ids, float* top_logprobs, void* workspace, size_t workspace_bytes, void* stream);

/* No-repeat-n-gram ban, in place, before b200_sample or b200_beam_search_step (Hugging Face no_repeat_ngram_size over the whole
 * history the caller passes; restated, parity with the reference's banRepeatNgram kernel unpinned). history [rows][hist_stride]
 * and hist_len [rows] as b200_sample takes them (hist_len is clamped to hist_stride). For row r with n = ngram_size[r] > 0 and
 * L = hist_len[r]: for every start s in [0, L - n] with h[s .. s+n-2] == h[L-n+1 .. L-1], logits[r][h[s+n-1]] = -inf (n == 1 bans
 * every token of the history); ids outside [0, vocab) are ignored; n <= 0 or L < n leaves the row alone. Every other logit keeps
 * its bits. logits dtype 0 fp16, 1 bf16, 2 fp32. Temperature, the penalties and b200_sample leave -inf at -inf, so the order of
 * this op and those does not matter. One CTA per row; under PDL it waits before reading anything. */
int b200_ban_repeat_ngram(void* logits, int dtype, int rows, int vocab, const int32_t* history, const int32_t* hist_len, int hist_stride,
                          const int32_t* ngram_size, void* stream);

/* Constrained decoding, in place on logits [rows][vocab] (dtype 0 fp16, 1 bf16, 2 fp32), before b200_argmax, b200_sample or
 * b200_beam_search_step: a grammar engine's token bitmask and OpenAI-style logit_bias.
 *   bitmask [rows][mask_stride] int32, xgrammar's layout: token t of row r is allowed iff (bitmask[r][t >> 5] >> (t & 31)) & 1
 *   (an all-ones word, -1, allows its 32 tokens); mask_stride >= ceil(vocab / 32); bits at t >= vocab are ignored; NULL = no
 *   mask. A masked token becomes the dtype's -inf and is never read.
 *   bias: a CSR over rows, bias_offsets [rows + 1] (offsets[0] = 0, non-decreasing) selects the entries [offsets[r],
 *   offsets[r+1]) of bias_ids / bias_values. An allowed token t = ids[e] becomes round_T(float(x) + values[e]): one fp32 add and
 *   one rounding to the logits' dtype (so fp16 can overflow to +-inf). Ids outside [0, vocab) are ignored, a bias on a masked
 *   token has no effect, and the ids of a row must be distinct (not checked). NULL bias_offsets = no bias.
 *   Every other logit keeps its bits, NaN included.
 * rows in 1..65535; at least one of bitmask and bias_offsets. A row whose mask allows nothing becomes all -inf: b200_argmax
 * then returns token 0, b200_sample token -1 with token_prob 0, and b200_beam_search_step scores the row's candidates -inf.
 * Cost: the mask pass reads rows * ceil(vocab / 32) words and writes only the masked tokens (a fully masked word as 16-byte
 * stores when the row is 16-byte aligned), so an all-ones mask writes nothing; only biased entries read logits. One launch,
 * deterministic, graph-capturable, recorded by decode programs; under PDL it writes nothing before its grid dependency. */
int b200_constrain_logits(void* logits, int dtype, int rows, int vocab, const int32_t* bitmask, int mask_stride,
                          const int32_t* bias_offsets, const int32_t* bias_ids, const float* bias_values, void* stream);

/* ------------------------------------------------------------------------------------------------ TP all-reduce over NVLink peer memory */

/* One-shot SUM all-reduce of a small [rows][hidden] fp16/bf16 tensor, the exchange after each row-parallel GEMM
 * (replaces all_reduce(t, Group.TP), rtp_llm/models_py/distributed/collective_torch.py:694-722; the reference's fast path
 * is torch symmetric memory, distributed/symm_mem.py:126-185). One process per GPU. Set-up, once per process:
 *   b200_peer_alloc(b200_peer_ar_region_bytes(max_msg), &mine, handle)  -> exchange the 64-byte handles between ranks
 *   (any host channel) -> b200_peer_open(handle_of_rank_r, &regions[r]) for r != rank; regions[rank] = mine.
 * Per call: every rank must issue the same sequence of peer_* calls on its stream. `call_parity` is ignored (kept for ABI
 * compatibility): the two data slots alternate by a device-side call counter, so CUDA graphs holding any number of calls
 * replay correctly. Deterministic: all ranks sum in rank order and get identical bits. A rank whose peers never arrive
 * traps after a few seconds of polling instead of hanging. bytes % 16 == 0, bytes <= max_message_bytes, world <= 8. */
size_t b200_peer_ar_region_bytes(size_t max_message_bytes);
int b200_peer_alloc(size_t bytes, void** ptr, void* ipc_handle_out);
int b200_peer_open(const void* ipc_handle, void** ptr);
int b200_peer_allreduce(const void* in, void* out, size_t bytes, int is_bf16, void* const* regions, size_t max_message_bytes,
                        int call_parity, int rank, int world, void* stream);

/* The same exchange fused with what follows it in the decoder layer: y = rmsnorm(allreduce(in) + residual) * gamma and
 * residual += allreduce(in), in ONE kernel (replaces all_reduce + fused_add_rmsnorm: collective_torch.py:694-722 then
 * RegisterBaseBindings.hpp:54; call sites hybrid/causal_attention.py:91-92, dense_mlp.py:104-105). Numerics are those of
 * the unfused sequence (the reduced value is rounded to the tensor type first). hidden % (8*world) == 0, hidden <= 8192. */
int b200_peer_allreduce_norm(const void* in, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                             float eps, void* const* regions, size_t max_message_bytes, int rank, int world, void* stream);

/* GEMM + reduce-scatter in ONE kernel, for the row-parallel GEMMs (o, w2) under tensor parallelism (reference sequence:
 * LinearBase.forward, then all_reduce(t, Group.TP): hybrid/causal_attention.py:90-92, dense_mlp.py:103-105). Same arguments
 * and arithmetic as b200_wo_gemm; the epilogue pushes every output element another rank owns (rank r owns the r-th 1/world
 * of the columns of every row) straight into that rank's reduce-scatter slot over NVLink while the tile is still in
 * registers; the columns this rank owns are stored to y. MUST be followed on the same stream by b200_peer_gather_norm over
 * the same y / regions with no other collective of this communicator in between (both derive the exchange epoch from the
 * communicator's device-side call counter). Bits are those of b200_wo_gemm + b200_peer_allreduce_norm.
 * N % 128 == 0, N % (8*world) == 0, N <= 8192, B*N*2 <= max_message_bytes, no SILU_MUL, not B200_FMT_INT4_G64 / _G32. */
int b200_wo_gemm_rs(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* col_scale,
                    const void* bias, void* y, void* workspace, size_t workspace_bytes, int flags, void* const* regions,
                    size_t max_message_bytes, int rank, int world, void* stream);
/* Second half of the fused exchange: reduce the own slice in rank order, all-gather, residual add, RMSNorm (the kernel of
 * b200_peer_allreduce_norm without its scatter phase, which the GEMM epilogue already did). */
int b200_peer_gather_norm(const void* in, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                          float eps, void* const* regions, size_t max_message_bytes, int rank, int world, void* stream);

/* Vocab-parallel greedy sampling: out[r] = argmax over the CONCATENATED vocabulary (rank r holds columns
 * [r*vocab_local, (r+1)*vocab_local), columns >= vocab_total are padding), lowest index on ties, identical on every rank.
 * Replaces the logits all-gather + argmax of cpp/models/PyWrappedModel.cc:915-936,1001-1052 for top_k == 1. */
int b200_peer_argmax(const void* logits, int is_bf16, int rows, int vocab_local, int vocab_total, int32_t* out,
                     void* const* regions, size_t max_message_bytes, int rank, int world, void* stream);

/* ------------------------------------------------------------------------------------------------ decode programs */

/* A decode program is a recorded sequence of the op calls above, replayed with far fewer launches -- this library's counterpart
 * of the reference's CUDA-graph capture of the decode step (rtp_llm/cpp/cuda_graph/cuda_graph_runner.cc: capture once per
 * batch size, replay every step).  Between b200_program_begin and b200_program_end every op call of the CALLING THREAD is
 * appended to the program instead of being launched.  Consecutive weight-only GEMMs, norms, rope+append, embedding and
 * block-table ops are fused into ONE persistent kernel (2 CTAs per SM, grid-wide barriers between ops, stream-K GEMMs,
 * weights prefetched across op boundaries -- csrc/decode_program.cuh); attention, FP16 GEMMs, argmax, sampling and
 * all-reduce calls keep their own launches, in order.  Everything an op call decides is decided when it is recorded and
 * never evaluated again by b200_program_launch: its argument checks, launch-shape plans and tensor maps, the B200_* test-hook
 * environment variables, and for the launches outside the persistent kernel the b200_set_pdl setting (the persistent
 * kernel's launches take the setting current at b200_program_launch; PDL never changes results).  Pointers and sizes are
 * frozen, exactly as under stream capture, and structs passed by pointer (b200_rope_config, the peer region array) are
 * copied, so the caller may reuse them.  b200_program_launch never allocates or synchronises and may itself be captured
 * into a CUDA graph.  b200_program_end allocates the device-side op table (once).
 * Results are identical to issuing the same calls one by one (same kernels' arithmetic; tests compare bit for bit). */
typedef struct b200_program b200_program;
int b200_program_create(b200_program** out);
int b200_program_begin(b200_program* p);
int b200_program_end(b200_program* p);
int b200_program_launch(b200_program* p, void* stream);
int b200_program_num_ops(const b200_program* p);      /* ops fused into persistent-kernel segments */
int b200_program_num_launches(const b200_program* p); /* kernel launches per b200_program_launch */
int b200_program_set_trace(b200_program* p, void* device_buffer); /* developer: per-op, per-CTA globaltimer stamps */
int b200_program_destroy(b200_program* p);

#ifdef __cplusplus
}
#endif
#endif /* B200_DECODE_OPS_H */
