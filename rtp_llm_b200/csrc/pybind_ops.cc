// pybind / torch face of the C ABI: the literal form of the reference's registration seam.
//
//   void rtp_llm::registerPyModuleOps(pybind11::module&)   == rtp_llm/models_py/bindings/RegisterOps.h:9 (one definition per
//        backend, chosen at link time by select_py_bindings(), arch_config/arch_select.bzl:189-201; the CUDA one is
//        cuda/RegisterCudaOps.cc:16). Linked into librtp_compute_ops.so it replaces that definition; built standalone (below) it is
//        the module `b200_compute_ops` with the same `rtp_llm_ops` submodule layout (cpp/pybind/ComputeInit.cc:25-26).
//   B200AttnOp    == XQAAttnOp (bindings/cuda/XQAAttnOp.{h:13-28,cc:52-176}): support / prepare / update /
//        update_kv_cache_offset / forward with the same argument meaning; XQAParams (CudaXqa.h:10-16) is mirrored as B200AttnParams.
//   B200LinearOp  == the compute behind a LinearBase strategy (linear_base.py:81) for weights packed by b200_pack_w4/w8.
// Inside the reference tree AttentionConfigs / PyAttentionInputs / LayerKVCache / ParamsBase are the reference's own types
// (cpp/model_utils/AttentionConfig.h:24-85, bindings/OpDefs.h:29-51,281-327, bindings/ParamsBase.h:8-22); standalone they are the
// minimal mirrors declared here (same member names). Only torch tensors and plain ints cross into include/b200_decode_ops.h.
#include <ATen/cuda/CUDAContext.h>
#include <cuda_runtime.h>
#include <torch/extension.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <string>

#include "../../include/b200_decode_ops.h"

namespace py = pybind11;

namespace rtp_llm {

// ---- error convention: RTP_LLM_CHECK_WITH_INFO -> exception -> Python RuntimeError (cpp/utils/AssertUtils.h:18-27)
#define B200_CHECK(cond, msg)                                  \
    do {                                                       \
        if (!(cond)) throw std::runtime_error(std::string(msg)); \
    } while (0)
static void check_rc(int rc, const char* what) {
    if (rc != 0) throw std::runtime_error(std::string(what) + " failed: " + b200_last_error());
}
static void* cur_stream() { return at::cuda::getCurrentCUDAStream(at::cuda::current_device()).stream(); }

// ---- standalone mirrors of the reference types (member names as in the reference)
// The RopeConfig fields the decode rope reads (cpp/model_utils/RopeConfig.h:21-42). The defaults are plain Base at base 10000
// over the whole head (dim 0 = size_per_head), which is what this seam computed before it read anything but `base`.
struct RopeConfig {
    int style = 1;   // RopeStyle: 0 No, 1 Base, 2 Glm2, 3 DynamicNTK, 4 QwenDynamicNTK, 5 Yarn, 6 Llama3, 7 Mrope
    int dim = 0;
    double base = 10000.0;
    double scale = 1.0;
    double factor1 = 0.0;
    double factor2 = 0.0;
    int max_pos = 0;
    double extrapolation_factor = 1.0;
    double mscale = 1.0;
    bool is_neox_style = true;
};
struct AttentionConfigs {
    size_t head_num = 0;
    size_t kv_head_num = 0;
    size_t size_per_head = 0;
    RopeConfig rope_config;
    size_t tokens_per_block = 8;
    size_t kernel_tokens_per_block = 0;
    float q_scaling = 1.0f;
    bool need_rope_kv_cache = true;
    bool use_logn_attn = false;
    bool kv_cache_fp8 = false;   // KvCacheDataType::FP8 in the reference
    size_t max_seq_len = 32768;
};
struct PyAttentionInputs {
    bool is_prefill = false;
    torch::Tensor sequence_lengths;                 // [B] int32, tokens already cached; CUDA or pinned host
    torch::Tensor kv_cache_kernel_block_id_device;  // [B, M] int32
    torch::Tensor input_lengths;                    // [B]: a verification step runs q_len = max(input_lengths) tokens per sequence
    torch::Tensor combo_position_ids;               // [B * q_len] int32 rotation positions (entries <= 0 keep the cache slot)
};
struct LayerKVCache {
    torch::Tensor kv_cache_base;  // [P, 2, Hkv, T, D]
    torch::Tensor kv_scale_base;  // unused (FP8 KV is out of scope)
};
class ParamsBase {
public:
    virtual ~ParamsBase() = default;
};
using ParamsBasePtr = std::shared_ptr<ParamsBase>;

struct B200AttnParams: public ParamsBase {
    size_t batch_size = 0;
    size_t max_seq_len = 0;
    size_t q_len = 1;                // query tokens per sequence (> 1: verification of speculative tokens)
    torch::Tensor kv_cache_offset;   // [B, 1, 2, M] int32
    torch::Tensor sequence_lengths;  // shares storage with the engine's tensor so graph replay can refresh it in place
    torch::Tensor position_ids;      // the inputs' combo_position_ids (undefined when absent)
    torch::Tensor workspace;
};
using B200AttnParamsPtr = std::shared_ptr<B200AttnParams>;

static size_t page_size_of(const AttentionConfigs& c) {
    return c.kernel_tokens_per_block ? c.kernel_tokens_per_block : c.tokens_per_block;
}

// == attention._q_len: max(input_lengths) when the inputs carry them, else 1
static size_t q_len_of(const PyAttentionInputs& in) {
    if (!in.input_lengths.defined() || in.input_lengths.numel() == 0) return 1;
    return (size_t)std::max<int64_t>(in.input_lengths.max().item<int64_t>(), 1);
}

static torch::Tensor position_ids_of(const PyAttentionInputs& in) {
    return in.combo_position_ids.defined() && in.combo_position_ids.numel() > 0 ? in.combo_position_ids : torch::Tensor();
}

// ---- the rope config, decided as rtp_llm_b200/rope.py decides it (the two seams serve the same configs with the same bits)
static int rotary_dim(const AttentionConfigs& c) { return c.rope_config.dim ? c.rope_config.dim : (int)c.size_per_head; }

static bool rope_supported(const AttentionConfigs& c) {
    const RopeConfig& r = c.rope_config;
    const int s = r.style, dim = rotary_dim(c);
    const bool served = s == 0 || s == 1 || s == 3 || s == 4 || s == 5 || s == 6;   // not Glm2 (2), Mrope (7) or unknown styles
    return served && r.is_neox_style && dim % 2 == 0 && dim > 0 && dim <= (int)c.size_per_head && (s == 0 || r.base > 1.0);
}

// Base over the whole head at scale 1 without logn or position ids: b200_rope_append(_multi), the bits of a base-only config
static bool rope_is_plain_base(const AttentionConfigs& c, bool has_position_ids) {
    const RopeConfig& r = c.rope_config;
    return r.style == 1 && r.scale == 1.0 && rotary_dim(c) == (int)c.size_per_head && r.is_neox_style && !c.use_logn_attn &&
           !has_position_ids;
}

// rope.build_table: the fp32 [int(max_pos * scale)][dim] interleaved (cos, sin) table of RopeCache.cc:16-85 for Base and Yarn,
// with the same ATen calls as the Python builder (so the same bits); undefined for other styles or an empty range.
static torch::Tensor build_rope_table(const RopeConfig& r, int dim) {
    const int64_t positions = (int64_t)(r.max_pos * r.scale);
    if ((r.style != 1 && r.style != 5) || positions <= 0) return torch::Tensor();
    const auto f32 = torch::kFloat;
    const torch::Tensor exps = torch::arange(0, dim, 2).to(f32) / dim;
    torch::Tensor freqs, cos, sin;
    if (r.style == 1) {
        const torch::Tensor inv_freq = torch::reciprocal(torch::pow(torch::scalar_tensor(r.base, f32), exps)) * 1.0;
        torch::Tensor t = torch::arange(positions).to(f32);
        t.div_(r.scale);
        freqs = torch::outer(t, inv_freq);
        cos = freqs.cos();
        sin = freqs.sin();
    } else {
        const torch::Tensor pos_freqs = torch::pow(torch::scalar_tensor(r.base, f32), exps);
        const torch::Tensor inv_e = torch::reciprocal(pos_freqs) * 1.0, inv_i = torch::reciprocal(pos_freqs * r.scale) * 1.0;
        auto corr = [&](double nrot) { return (double)dim * std::log(r.max_pos / (nrot * 2.0 * M_PI)) / (2.0 * std::log(r.base)); };
        const double low = (double)std::max(0, (int)std::floor(corr(r.factor1)));
        double high = (double)std::min(dim - 1, (int)std::ceil(corr(r.factor2)));
        if (std::abs(low - high) < 1e-6) high += 0.001;
        const torch::Tensor ramp = torch::clamp((torch::arange(dim / 2).to(f32) - low) / (high - low), 0, 1);
        const torch::Tensor mask = torch::rsub(ramp, 1.0) * r.extrapolation_factor;
        const torch::Tensor inv_freq = inv_i * torch::rsub(mask, 1.0) + inv_e * mask;
        freqs = torch::outer(torch::arange(positions).to(f32), inv_freq);
        cos = freqs.cos() * r.mscale;
        sin = freqs.sin() * r.mscale;
    }
    return torch::stack({cos, sin}, -1).reshape({positions, -1}).contiguous();
}

// rope.table: built and uploaded once per (config, device)
static torch::Tensor rope_table(const RopeConfig& r, int dim, const torch::Device& device) {
    static std::mutex mu;
    static std::map<std::string, torch::Tensor> tables;
    char key[256];
    snprintf(key, sizeof(key), "%d %d %a %a %a %a %d %a %a %s", r.style, dim, r.base, r.scale, r.factor1, r.factor2, r.max_pos,
             r.extrapolation_factor, r.mscale, device.str().c_str());
    std::lock_guard<std::mutex> lock(mu);
    auto it = tables.find(key);
    if (it == tables.end()) {
        torch::Tensor t = build_rope_table(r, dim);
        it = tables.emplace(key, t.defined() ? t.to(device) : t).first;
    }
    return it->second;
}

// == ops.check_lengths: the sequence lengths a kernel reads through their pointer are int32, contiguous, at least `seqs` long, and
// in device or pinned host memory. A pageable host tensor would hand the kernel a host pointer, an int64 one pairs of int32.
static void check_lengths(const torch::Tensor& t, int64_t seqs, const char* who) {
    B200_CHECK(t.defined() && t.scalar_type() == torch::kInt32 && t.is_contiguous() && t.numel() >= seqs &&
                   (t.is_cuda() || t.is_pinned()),
               std::string(who) + ": sequence_lengths must be a contiguous int32 tensor of at least " + std::to_string(seqs) +
                   " entries in CUDA or pinned host memory");
}

static void update_offset_tensor(const torch::Tensor& kv_cache_offset, const torch::Tensor& block_ids) {
    B200_CHECK(block_ids.defined() && block_ids.is_cuda() && block_ids.scalar_type() == torch::kInt32 && block_ids.dim() == 2,
               "B200AttnOp expects a CUDA int32 block table [batch, blocks]");
    B200_CHECK(kv_cache_offset.scalar_type() == torch::kInt32, "B200AttnOp expects int32 kv_cache_offset");
    B200_CHECK(kv_cache_offset.dim() == 4 && kv_cache_offset.size(1) == 1 && kv_cache_offset.size(2) == 2,
               "B200AttnOp expects kv_cache_offset shape [batch, 1, 2, blocks]");
    B200_CHECK(kv_cache_offset.size(0) == block_ids.size(0) && kv_cache_offset.size(3) == block_ids.size(1),
               "B200AttnOp shape mismatch: offset vs block table");
    check_rc(b200_convert_block_table(kv_cache_offset.data_ptr<int>(), block_ids.data_ptr<int>(), (int)block_ids.size(0),
                                      (int)block_ids.size(1), cur_stream()),
             "b200_convert_block_table");
}

class B200AttnOp {
public:
    explicit B200AttnOp(const AttentionConfigs& attn_configs): attn_configs_(attn_configs) {}

    // group * q_len <= 64 query rows per (sequence, kv head); when this seam applies the rope, the rope config must be served
    // (attention.B200DecodeImpl.support applies the same rule), so an engine falls through to another op instead
    bool support(PyAttentionInputs attn_inputs) {
        const auto& c = attn_configs_;
        if (attn_inputs.is_prefill || c.kv_cache_fp8 || c.kv_head_num == 0 || c.head_num % c.kv_head_num) return false;
        if (c.need_rope_kv_cache && !rope_supported(c)) return false;
        const size_t group = c.head_num / c.kv_head_num, T = page_size_of(c);
        if ((c.size_per_head != 64 && c.size_per_head != 128 && c.size_per_head != 256) || group < 1 ||
            group * q_len_of(attn_inputs) > 64)
            return false;
        if (!(T == 16 || T == 32 || T == 64 || T == 128)) return false;
        return b200_device_check(at::cuda::current_device()) == 0;
    }

    ParamsBasePtr prepare(PyAttentionInputs attn_inputs) {
        auto params = std::make_shared<B200AttnParams>();
        const auto& block_ids = attn_inputs.kv_cache_kernel_block_id_device;
        B200_CHECK(block_ids.defined(), "decode should have kv cache block id.");
        check_lengths(attn_inputs.sequence_lengths, block_ids.size(0), "B200AttnOp::prepare");
        const int64_t batch = attn_inputs.sequence_lengths.numel();
        B200_CHECK(block_ids.size(0) == batch, "kv blocks batch size does not match sequence_lengths");
        params->kv_cache_offset = torch::empty({batch, 1, 2, block_ids.size(1)}, block_ids.options());
        update_offset_tensor(params->kv_cache_offset, block_ids);
        params->batch_size = (size_t)batch;
        params->q_len = q_len_of(attn_inputs);
        // XQAAttnOp.cc:147-149 passes max_seq_len + 1; with q_len tokens per sequence the bound is max_seq_len + q_len
        const size_t cap = (size_t)block_ids.size(1) * page_size_of(attn_configs_), want = attn_configs_.max_seq_len + params->q_len;
        params->max_seq_len = want < cap ? want : cap;
        params->sequence_lengths = attn_inputs.sequence_lengths;
        params->position_ids = position_ids_of(attn_inputs);
        const size_t ws = b200_paged_decode_attn_workspace_bytes(params->batch_size * params->q_len, attn_configs_.head_num,
                                                                 attn_configs_.kv_head_num, params->max_seq_len);
        params->workspace = torch::zeros({(int64_t)(ws ? ws : 256)}, torch::TensorOptions().dtype(torch::kUInt8).device(block_ids.device()));
        if (attn_configs_.need_rope_kv_cache)   // the cos/sin table is uploaded here, never inside a graph capture
            rope_table(attn_configs_.rope_config, rotary_dim(attn_configs_), block_ids.device());
        return params;
    }

    void update(const B200AttnParamsPtr& params, PyAttentionInputs attn_inputs) {
        B200_CHECK(params != nullptr, "B200AttnOp::update received null params");
        B200_CHECK(attn_inputs.kv_cache_kernel_block_id_device.defined(), "decode should have kv cache block id.");
        check_lengths(attn_inputs.sequence_lengths, attn_inputs.kv_cache_kernel_block_id_device.size(0), "B200AttnOp::update");
        update_offset_tensor(params->kv_cache_offset, attn_inputs.kv_cache_kernel_block_id_device);
        params->batch_size = (size_t)attn_inputs.kv_cache_kernel_block_id_device.size(0);
        params->sequence_lengths = attn_inputs.sequence_lengths;
        params->position_ids = position_ids_of(attn_inputs);
    }

    void updateKvCacheOffset(const torch::Tensor& kv_cache_offset, const torch::Tensor& kv_cache_block_id_device) {
        update_offset_tensor(kv_cache_offset, kv_cache_block_id_device);
    }

    torch::Tensor forward(const torch::Tensor& input, std::optional<LayerKVCache> kv_cache, const B200AttnParamsPtr& params) {
        B200_CHECK(kv_cache.has_value(), "decode should have kv cache.");
        B200_CHECK(params != nullptr, "B200AttnOp::forward received null params");
        check_lengths(params->sequence_lengths, (int64_t)params->batch_size, "B200AttnOp::forward");
        const auto& c = attn_configs_;
        const int64_t rows = input.size(0);
        torch::Tensor out = torch::empty({rows, (int64_t)(c.head_num * c.size_per_head)}, input.options());
        const auto& pool = kv_cache->kv_cache_base;
        const int is_bf16 = input.scalar_type() == torch::kBFloat16;
        const auto* seq = reinterpret_cast<const uint32_t*>(params->sequence_lengths.data_ptr());
        if (params->q_len > 1) {   // input [B*q_len, Hq*D] token-major == q [B][q_len][Hq][D]; out [B*q_len, Hq*D]
            B200_CHECK(rows == (int64_t)(params->batch_size * params->q_len), "B200AttnOp: input rows must be batch x q_len");
            check_rc(b200_paged_decode_attn_multi(input.data_ptr(), is_bf16, out.data_ptr(), c.head_num, c.kv_head_num, c.size_per_head,
                                                  params->batch_size, params->q_len, (size_t)params->kv_cache_offset.size(3),
                                                  params->max_seq_len, page_size_of(c), pool.data_ptr(),
                                                  params->kv_cache_offset.data_ptr<int>(), seq, 1.0f / c.q_scaling,
                                                  params->workspace.data_ptr(), (size_t)params->workspace.numel(), cur_stream()),
                     "b200_paged_decode_attn_multi");
            return out;
        }
        check_rc(b200_paged_decode_attn(input.data_ptr(), is_bf16, out.data_ptr(), c.head_num, c.kv_head_num, c.size_per_head,
                                        params->batch_size, (size_t)params->kv_cache_offset.size(3), params->max_seq_len,
                                        page_size_of(c), pool.data_ptr(), params->kv_cache_offset.data_ptr<int>(), seq,
                                        1.0f / c.q_scaling, params->workspace.data_ptr(), (size_t)params->workspace.numel(),
                                        cur_stream()),
                 "b200_paged_decode_attn");
        return out;
    }

private:
    AttentionConfigs attn_configs_;
};

// rope + append: FusedRopeKVCacheDecodeOp.forward (rtp_llm/ops/fused_rope_kvcache_op.py:202-246). qkv [B*q_len, (Hq+2Hkv)*D]
// token-major, q_len from the params; returns q [B*q_len, Hq*D]. A plain Base config without logn or position ids runs
// b200_rope_append(_multi); every other served config runs b200_rope_append_ex(_multi), with the cos/sin table for Base and Yarn.
static torch::Tensor b200_rope_kvcache_decode(const torch::Tensor& qkv, const LayerKVCache& kv_cache, const B200AttnParamsPtr& params,
                                              const AttentionConfigs& c) {
    B200_CHECK(params != nullptr, "b200_rope_kvcache_decode received null params");
    B200_CHECK(rope_supported(c), "b200_rope_kvcache_decode: rope config not served (style / pairing / rotary dim)");
    const auto& pool = kv_cache.kv_cache_base;
    const int q_len = (int)params->q_len, rows = (int)qkv.size(0), is_bf16 = qkv.scalar_type() == torch::kBFloat16;
    B200_CHECK(q_len >= 1 && rows % q_len == 0, "b200_rope_kvcache_decode: qkv rows must be a multiple of q_len");
    check_lengths(params->sequence_lengths, rows / q_len, "b200_rope_kvcache_decode");
    torch::Tensor q = torch::empty({qkv.size(0), (int64_t)(c.head_num * c.size_per_head)}, qkv.options());
    const int32_t* seq = params->sequence_lengths.data_ptr<int>();
    const int M = (int)params->kv_cache_offset.size(3), T = (int)page_size_of(c);
    torch::Tensor pid = params->position_ids;
    if (rope_is_plain_base(c, pid.defined())) {
        if (q_len == 1)
            check_rc(b200_rope_append(qkv.data_ptr(), q.data_ptr(), pool.data_ptr(), params->kv_cache_offset.data_ptr<int>(), seq,
                                      is_bf16, rows, (int)c.head_num, (int)c.kv_head_num, (int)c.size_per_head, M, T,
                                      (float)c.rope_config.base, cur_stream()),
                     "b200_rope_append");
        else
            check_rc(b200_rope_append_multi(qkv.data_ptr(), q.data_ptr(), pool.data_ptr(), params->kv_cache_offset.data_ptr<int>(), seq,
                                            is_bf16, rows / q_len, (int)c.head_num, (int)c.kv_head_num, (int)c.size_per_head, M, T,
                                            (float)c.rope_config.base, q_len, cur_stream()),
                     "b200_rope_append_multi");
        return q;
    }
    if (pid.defined()) {
        B200_CHECK(pid.numel() == rows, "b200_rope_kvcache_decode: combo_position_ids needs one entry per qkv row");
        pid = pid.to(qkv.device(), torch::kInt32).contiguous();
    }
    const RopeConfig& r = c.rope_config;
    const b200_rope_config cfg{r.style, rotary_dim(c), (float)r.base, (float)r.scale, (float)r.factor1, (float)r.factor2, r.max_pos,
                               (float)r.extrapolation_factor, (float)r.mscale};
    const torch::Tensor table = rope_table(r, cfg.dim, qkv.device());
    const float* cache = table.defined() ? table.data_ptr<float>() : nullptr;
    const int cache_positions = table.defined() ? (int)table.size(0) : 0;
    const int32_t* pids = pid.defined() ? pid.data_ptr<int>() : nullptr;
    if (q_len == 1)
        check_rc(b200_rope_append_ex(qkv.data_ptr(), nullptr, q.data_ptr(), pool.data_ptr(), params->kv_cache_offset.data_ptr<int>(),
                                     seq, pids, cache, cache_positions, &cfg, c.use_logn_attn, is_bf16, rows, (int)c.head_num,
                                     (int)c.kv_head_num, (int)c.size_per_head, M, T, cur_stream()),
                 "b200_rope_append_ex");
    else
        check_rc(b200_rope_append_ex_multi(qkv.data_ptr(), nullptr, q.data_ptr(), pool.data_ptr(),
                                           params->kv_cache_offset.data_ptr<int>(), seq, pids, cache, cache_positions, &cfg,
                                           c.use_logn_attn, is_bf16, rows / q_len, (int)c.head_num, (int)c.kv_head_num,
                                           (int)c.size_per_head, M, T, q_len, cur_stream()),
                 "b200_rope_append_ex_multi");
    return q;
}

// Y = X . W' for a weight already in the b200 blob layout (b200_pack_w4 / w8) or [N, K] fp16
class B200LinearOp {
public:
    B200LinearOp(int fmt, int64_t K, int64_t N, torch::Tensor weight, std::optional<torch::Tensor> col_scale,
                 std::optional<torch::Tensor> bias):
        fmt_(fmt), K_(K), N_(N), weight_(std::move(weight)), col_scale_(std::move(col_scale)), bias_(std::move(bias)) {
        const size_t ws = b200_wo_gemm_workspace_bytes(128, (int)N, (int)K);
        workspace_ = torch::zeros({(int64_t)(ws ? ws : 256)}, torch::TensorOptions().dtype(torch::kUInt8).device(weight_.device()));
    }
    torch::Tensor forward(const torch::Tensor& input) {
        B200_CHECK(input.dim() == 2 && input.size(1) == K_ && input.is_contiguous(), "B200LinearOp expects contiguous [B, K] input");
        torch::Tensor out = torch::empty({input.size(0), N_}, input.options());
        for (int64_t b0 = 0; b0 < input.size(0); b0 += 128) {
            const int64_t nb = std::min<int64_t>(128, input.size(0) - b0);
            check_rc(b200_wo_gemm(fmt_, input.scalar_type() == torch::kBFloat16, input[b0].data_ptr(), (int)nb, (int)K_, (int)N_,
                                  weight_.data_ptr(), col_scale_ ? col_scale_->data_ptr() : nullptr, bias_ ? bias_->data_ptr() : nullptr,
                                  out[b0].data_ptr(), workspace_.data_ptr(), (size_t)workspace_.numel(), 0, cur_stream()),
                     "b200_wo_gemm");
        }
        return out;
    }

private:
    int fmt_;
    int64_t K_, N_;
    torch::Tensor weight_, workspace_;
    std::optional<torch::Tensor> col_scale_, bias_;
};

// ---- glue ops under the reference's own names and argument lists (registerBasicCudaOps, cuda/RegisterBaseBindings.hpp:45-160;
// prototypes 3rdparty/flashinfer/flashinfer.h:21-31, common/FusedQKRmsNorm.cc:17-25, common/RtpEmbeddingLookup.cc:14-19): a model file
// that calls rtp_llm_ops.rmsnorm / fused_add_rmsnorm / silu_and_mul / fused_qk_rmsnorm / embedding runs unchanged on this plugin.
// cuda_stream: the raw stream handle the callers pass (torch.cuda.current_stream().cuda_stream, modules/base/cuda/norm.py:22); 0 = current.
static void* stream_arg(int64_t cuda_stream) { return cuda_stream ? reinterpret_cast<void*>(cuda_stream) : cur_stream(); }
static void check_rows(const torch::Tensor& t, const char* what) {
    B200_CHECK(t.defined() && t.is_cuda() && t.is_contiguous() && t.dim() == 2, std::string(what) + ": expected a contiguous 2-D CUDA tensor");
    B200_CHECK(t.scalar_type() == torch::kFloat16 || t.scalar_type() == torch::kBFloat16, std::string(what) + ": expected fp16 / bf16");
}

static void rmsnorm(torch::Tensor& output, torch::Tensor& input, torch::Tensor& weight, double eps, int64_t cuda_stream) {
    check_rows(input, "rmsnorm input");
    check_rows(output, "rmsnorm output");
    B200_CHECK(output.sizes() == input.sizes() && weight.numel() == input.size(1) && weight.scalar_type() == input.scalar_type(),
               "rmsnorm: shape / dtype mismatch");
    check_rc(b200_add_rmsnorm(input.data_ptr(), nullptr, weight.data_ptr(), output.data_ptr(), input.scalar_type() == torch::kBFloat16,
                              (int)input.size(0), (int)input.size(1), (float)eps, stream_arg(cuda_stream)),
             "b200_add_rmsnorm");
}

// flashinfer semantics: residual <- input + residual (rounded to the tensor type), input <- rmsnorm(unrounded sum) * weight
static void fused_add_rmsnorm(torch::Tensor& input, torch::Tensor& residual, torch::Tensor& weight, double eps, int64_t cuda_stream) {
    check_rows(input, "fused_add_rmsnorm input");
    check_rows(residual, "fused_add_rmsnorm residual");
    B200_CHECK(residual.sizes() == input.sizes() && weight.numel() == input.size(1) && weight.scalar_type() == input.scalar_type() &&
                   residual.scalar_type() == input.scalar_type(),
               "fused_add_rmsnorm: shape / dtype mismatch");
    torch::Tensor out = torch::empty_like(input);      // the kernel's input and output do not alias; the result is copied back in stream order
    void* st = stream_arg(cuda_stream);
    check_rc(b200_add_rmsnorm(input.data_ptr(), residual.data_ptr(), weight.data_ptr(), out.data_ptr(),
                              input.scalar_type() == torch::kBFloat16, (int)input.size(0), (int)input.size(1), (float)eps, st),
             "b200_add_rmsnorm");
    B200_CHECK(cudaMemcpyAsync(input.data_ptr(), out.data_ptr(), (size_t)input.numel() * input.element_size(), cudaMemcpyDeviceToDevice,
                               reinterpret_cast<cudaStream_t>(st)) == cudaSuccess,
               "fused_add_rmsnorm: copy back failed");
}

static void silu_and_mul(torch::Tensor& output, torch::Tensor& input, int64_t cuda_stream) {
    check_rows(input, "silu_and_mul input");
    check_rows(output, "silu_and_mul output");
    B200_CHECK(input.size(1) % 2 == 0 && output.size(0) == input.size(0) && output.size(1) * 2 == input.size(1) &&
                   output.scalar_type() == input.scalar_type(),
               "silu_and_mul: expected input [rows, 2*inter] (gate | up) and output [rows, inter]");
    check_rc(b200_silu_and_mul(input.data_ptr(), output.data_ptr(), input.scalar_type() == torch::kBFloat16, (int)input.size(0),
                               (int)(input.size(1) / 2), stream_arg(cuda_stream)),
             "b200_silu_and_mul");
}

// in place on IO [m, n] = rows of q heads | k heads | v heads; q_group_num / k_group_num = head counts, norm_size = head size
static void fused_qk_rmsnorm(torch::Tensor& IO, torch::Tensor& q_gamma, torch::Tensor& k_gamma, double layernorm_eps, int64_t q_group_num,
                             int64_t k_group_num, int64_t m, int64_t n, int64_t norm_size) {
    check_rows(IO, "fused_qk_rmsnorm IO");
    B200_CHECK(IO.size(0) == m && IO.size(1) == n && n == (q_group_num + 2 * k_group_num) * norm_size,
               "fused_qk_rmsnorm: n must equal (q_group_num + 2 * k_group_num) * norm_size");
    B200_CHECK(q_gamma.numel() == norm_size && k_gamma.numel() == norm_size && q_gamma.scalar_type() == IO.scalar_type() &&
                   k_gamma.scalar_type() == IO.scalar_type(),
               "fused_qk_rmsnorm: gamma shape / dtype mismatch");
    check_rc(b200_qk_rmsnorm(IO.data_ptr(), q_gamma.data_ptr(), k_gamma.data_ptr(), nullptr, nullptr, IO.scalar_type() == torch::kBFloat16,
                             (int)m, (int)q_group_num, (int)k_group_num, (int)norm_size, (float)layernorm_eps, cur_stream()),
             "b200_qk_rmsnorm");
}

static void embedding(torch::Tensor& output, torch::Tensor& input, torch::Tensor& weight, std::optional<torch::Tensor> position_ids,
                      std::optional<torch::Tensor> token_type_ids, std::optional<torch::Tensor> text_tokens_mask) {
    auto given = [](const std::optional<torch::Tensor>& t) { return t.has_value() && t->defined() && t->numel() > 0; };
    B200_CHECK(!given(position_ids) && !given(token_type_ids) && !given(text_tokens_mask),
               "embedding: position / token-type / mask tables are outside the decode path built here");
    B200_CHECK(input.is_cuda() && input.is_contiguous() && input.dim() == 1 && input.scalar_type() == torch::kInt32,
               "embedding: expected contiguous int32 token ids [tokens]");
    check_rows(weight, "embedding weight");
    check_rows(output, "embedding output");
    B200_CHECK(output.size(0) == input.size(0) && output.size(1) == weight.size(1) && output.scalar_type() == weight.scalar_type(),
               "embedding: output must be [tokens, hidden] of the weight's type");
    check_rc(b200_embedding(input.data_ptr<int>(), weight.data_ptr(), output.data_ptr(), weight.scalar_type() == torch::kBFloat16,
                            (int)input.size(0), (int)weight.size(1), cur_stream()),
             "b200_embedding");
}

void registerPyModuleOps(pybind11::module& m) {
    m.def("rmsnorm", &rmsnorm, "RMSNorm kernel", py::arg("output"), py::arg("input"), py::arg("weight"), py::arg("eps"),
          py::arg("cuda_stream") = 0);
    m.def("fused_add_rmsnorm", &fused_add_rmsnorm, "Fused Add RMSNorm kernel", py::arg("input"), py::arg("residual"), py::arg("weight"),
          py::arg("eps"), py::arg("cuda_stream") = 0);
    m.def("silu_and_mul", &silu_and_mul, "SiLU and Multiply kernel", py::arg("output"), py::arg("input"), py::arg("cuda_stream") = 0);
    m.def("fused_qk_rmsnorm", &fused_qk_rmsnorm, "Fused QK RMSNorm kernel", py::arg("IO"), py::arg("q_gamma"), py::arg("k_gamma"),
          py::arg("layernorm_eps"), py::arg("q_group_num"), py::arg("k_group_num"), py::arg("m"), py::arg("n"), py::arg("norm_size"));
    m.def("embedding", &embedding, "Embedding lookup kernel", py::arg("output"), py::arg("input"), py::arg("weight"),
          py::arg("position_ids") = py::none(), py::arg("token_type_ids") = py::none(), py::arg("text_tokens_mask") = py::none());
    py::class_<RopeConfig>(m, "RopeConfig")
        .def(py::init<>())
        .def_readwrite("style", &RopeConfig::style)
        .def_readwrite("dim", &RopeConfig::dim)
        .def_readwrite("base", &RopeConfig::base)
        .def_readwrite("scale", &RopeConfig::scale)
        .def_readwrite("factor1", &RopeConfig::factor1)
        .def_readwrite("factor2", &RopeConfig::factor2)
        .def_readwrite("max_pos", &RopeConfig::max_pos)
        .def_readwrite("extrapolation_factor", &RopeConfig::extrapolation_factor)
        .def_readwrite("mscale", &RopeConfig::mscale)
        .def_readwrite("is_neox_style", &RopeConfig::is_neox_style);
    py::class_<AttentionConfigs>(m, "AttentionConfigs")
        .def(py::init<>())
        .def_readwrite("head_num", &AttentionConfigs::head_num)
        .def_readwrite("kv_head_num", &AttentionConfigs::kv_head_num)
        .def_readwrite("size_per_head", &AttentionConfigs::size_per_head)
        .def_readwrite("rope_config", &AttentionConfigs::rope_config)
        .def_readwrite("tokens_per_block", &AttentionConfigs::tokens_per_block)
        .def_readwrite("kernel_tokens_per_block", &AttentionConfigs::kernel_tokens_per_block)
        .def_readwrite("q_scaling", &AttentionConfigs::q_scaling)
        .def_readwrite("need_rope_kv_cache", &AttentionConfigs::need_rope_kv_cache)
        .def_readwrite("use_logn_attn", &AttentionConfigs::use_logn_attn)
        .def_readwrite("kv_cache_fp8", &AttentionConfigs::kv_cache_fp8)
        .def_readwrite("max_seq_len", &AttentionConfigs::max_seq_len);
    py::class_<PyAttentionInputs>(m, "PyAttentionInputs")
        .def(py::init<>())
        .def_readwrite("is_prefill", &PyAttentionInputs::is_prefill)
        .def_readwrite("sequence_lengths", &PyAttentionInputs::sequence_lengths)
        .def_readwrite("kv_cache_kernel_block_id_device", &PyAttentionInputs::kv_cache_kernel_block_id_device)
        .def_readwrite("input_lengths", &PyAttentionInputs::input_lengths)
        .def_readwrite("combo_position_ids", &PyAttentionInputs::combo_position_ids);
    py::class_<LayerKVCache>(m, "LayerKVCache")
        .def(py::init<>())
        .def_readwrite("kv_cache_base", &LayerKVCache::kv_cache_base)
        .def_readwrite("kv_scale_base", &LayerKVCache::kv_scale_base);
    py::class_<ParamsBase, ParamsBasePtr>(m, "ParamsBase");
    py::class_<B200AttnParams, B200AttnParamsPtr, ParamsBase>(m, "B200AttnParams")
        .def(py::init<>())
        .def("__cpp_ptr__", [](B200AttnParams& self) { return reinterpret_cast<uintptr_t>(&self); }, "Get C++ object pointer address")
        .def_readwrite("kv_cache_offset", &B200AttnParams::kv_cache_offset)
        .def_readonly("q_len", &B200AttnParams::q_len);
    // same .def list as registerXQAAttnOp (XQAAttnOp.cc:158-176)
    py::class_<B200AttnOp>(m, "B200AttnOp")
        .def(py::init<const AttentionConfigs&>(), py::arg("attn_configs"))
        .def("support", &B200AttnOp::support, py::arg("attn_inputs").noconvert())
        .def("prepare", &B200AttnOp::prepare, py::arg("attn_inputs"))
        .def("update", &B200AttnOp::update, py::arg("params"), py::arg("attn_inputs"))
        .def("update_kv_cache_offset", &B200AttnOp::updateKvCacheOffset, py::arg("kv_cache_offset"),
             py::arg("kv_cache_block_id_device"))
        .def("forward", &B200AttnOp::forward, py::arg("input"), py::arg("kv_cache"), py::arg("params"));
    m.def("b200_rope_kvcache_decode", &b200_rope_kvcache_decode, py::arg("qkv"), py::arg("kv_cache"), py::arg("params"),
          py::arg("attn_configs"));
    py::class_<B200LinearOp>(m, "B200LinearOp")
        .def(py::init<int, int64_t, int64_t, torch::Tensor, std::optional<torch::Tensor>, std::optional<torch::Tensor>>(),
             py::arg("fmt"), py::arg("K"), py::arg("N"), py::arg("weight"), py::arg("col_scale") = std::nullopt,
             py::arg("bias") = std::nullopt)
        .def("forward", &B200LinearOp::forward, py::arg("input"));
}

}  // namespace rtp_llm

// standalone plugin form: module `b200_compute_ops` with the `rtp_llm_ops` submodule (cpp/pybind/ComputeInit.cc:18-27)
PYBIND11_MODULE(b200_compute_ops, m) {
    m.doc() = "Hopper-native decode ops behind rtp-llm's registerPyModuleOps seam";
    auto ops = m.def_submodule("rtp_llm_ops", "rtp llm custom ops (Hopper decode path)");
    rtp_llm::registerPyModuleOps(ops);
}
