// C-ABI entry points of libb200_decode.so (declared in include/b200_decode_ops.h).
// Host side only: argument checks, tensor-map encoding, launch-shape heuristics, launches, and the recorder that turns a
// sequence of op calls into a decode program (b200_program_*). No torch, no allocation on the op path.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "aux_kernels.cuh"
#include "decode_program.cuh"
#include "internal.h"
#include "paged_decode_attn.cuh"
#include "peer_allreduce.cuh"
#include "sampling.cuh"
#include "wo_gemm.cuh"

using namespace b200;
using namespace b200_host;

namespace b200_host {

thread_local std::string g_err;
thread_local unsigned long long* g_ftrace_next = nullptr;
static std::atomic<uint64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

int launched(const char* what) {
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(B200_ECUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return B200_OK;
}

// The library reads three environment variables, all test hooks that force one parameter of a launch plan the plan could
// also pick itself, so that tests reach every cluster size and the two-shot all-reduce deterministically:
// B200_ATTN_TILES_PER_SPLIT (attention split), B200_GEMM_SPLITK (cluster GEMM split-K) and B200_AR_TWOSHOT (all-reduce).
int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

int num_sms() {
    static int sms[16] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 16) return 132;
    if (!sms[dev]) {
        cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
        if (sms[dev] <= 0) sms[dev] = 132;   // no device (host-only planning): an H100 SXM
    }
    return sms[dev];
}

}  // namespace b200_host

namespace {

std::atomic<int> g_pdl{0};

// ---- cuTensorMapEncodeTiled through the runtime (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int make_map(CUtensorMap* map, bool bf16, int rank, const void* base, const cuuint64_t* dims,
             const cuuint64_t* strides_bytes /*rank-1*/, const cuuint32_t* box) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return fail(B200_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank,
                    const_cast<void*>(base), dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(B200_ECUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return B200_OK;
}

size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- attention launch shape
constexpr int kAttnMaxSplit = 64;
void attn_split(int units, int max_tiles, int* nsplit, int* tiles_per_split, int head_dim = 128) {
    int forced = env_int("B200_ATTN_TILES_PER_SPLIT", 0);
    int best_c = max_tiles;
    double best = 1e30;
    const int sms = num_sms();
    // Cost model (not refitted on H100; hbm = what an H100 SXM's 3.35 TB/s HBM3 sustains in practice): a CTA has ~3 us of
    // fixed time, streams its 32 KB tiles at min(60 GB/s -- what its 96 KB ring sustains --, HBM / resident CTAs), CTAs
    // beyond 2*SMs are back-filled (fractional waves), a split adds ~3 us of merge.
    const double slots = 2.0 * sms, hbm = 3.0e12, r_cta = 60e9, fixed = 3e-6, merge = 3e-6, tile_bytes = 32768.0 * head_dim / 128.0;
    for (int c = 1; c <= max_tiles; ++c) {
        const int ns = (max_tiles + c - 1) / c;
        if (ns > kAttnMaxSplit) continue;
        const double ctas = (double)units * ns;
        const double waves = std::max(1.0, ctas / slots);   // beyond one wave CTAs are back-filled, not lock-stepped
        const double resident = ctas < slots ? ctas : slots;
        const double rate = std::min(r_cta, hbm / resident);
        // merging the splits: <= 8 splits form a cluster and merge through DSMEM (~1.5 us); more go through the L2 workspace and
        // a last-arriver loop whose cost grows with the split count (measured 26 us for 16 splits x 8 tiles, r02)
        const double merge_cost = ns == 1 ? 0.0 : (ns <= 8 ? 1.5e-6 : merge + 0.55e-6 * ns);
        const double cost = waves * (fixed + c * tile_bytes / rate) + merge_cost;
        if (cost < best * (1.0 - 1e-6) || (std::fabs(cost - best) <= best * 1e-6 && c > best_c)) {
            best = cost;
            best_c = c;
        }
    }
    if (forced > 0) best_c = forced < max_tiles ? forced : max_tiles;
    int ns = (max_tiles + best_c - 1) / best_c;
    if (ns > kAttnMaxSplit) {
        ns = kAttnMaxSplit;
        best_c = (max_tiles + ns - 1) / ns;
        ns = (max_tiles + best_c - 1) / best_c;
    }
    *nsplit = ns;
    *tiles_per_split = best_c;
}

// Workspace of a launch whose splits merge through L2 (more than 8 splits): [sem][ml][o], one counter per (sequence, kv head),
// then a running max / sum and a partial output per (query row, split).
struct AttnWorkspace {
    size_t sem, ml, o;
};
AttnWorkspace attn_workspace(size_t batch, size_t head_num, size_t kv_head_num, size_t q_len, size_t nsplit, size_t head_dim) {
    const size_t slots = batch * head_num * q_len * nsplit;
    return {round_up(batch * kv_head_num * sizeof(int), 256), round_up(slots * 2 * sizeof(float), 256),
            slots * head_dim * sizeof(float)};
}

// ---- GEMM launch shape
int gemm_bpad(int B) { return B <= 16 ? 16 : (B <= 32 ? 32 : (B <= 64 ? 64 : 128)); }
// one-kernel-per-GEMM path (gemm_cluster.cu): split-K so that one wave of 2*SMs CTAs is filled. The nsplit CTAs of a tile
// merge their partials through L2 (at most 8 slots; the reduce-scatter GEMM merges them in a thread-block cluster, and 8 is
// the portable cluster size). The GPC rule below stays from the cluster merge, which needs a cluster's CTAs in one GPC: it
// keeps the plan of the two merges the same, so the reduce-scatter GEMM and the plain one give the same bits.
constexpr int kGemmMaxSplit = 8;
void gemm_split(int n_tiles, int k_blocks, int* nsplit, int* kb_per_split) {
    const int forced = env_int("B200_GEMM_SPLITK", 0);
    const long slots = 2L * num_sms();
    int best_s = 1;
    double best = 1e30;
    const int smax = k_blocks < kGemmMaxSplit ? k_blocks : kGemmMaxSplit;
    for (int s = 1; s <= smax; ++s) {
        if (s > 1 && n_tiles >= slots) break;   // already more than a wave of tiles: splitting only adds merge traffic
        if (s > 1 && (s & (s - 1))) continue;                       // powers of two pack GPCs without strays
        if (s > 1 && n_tiles > 8 * (32 / s)) continue;              // >= 16 SMs (32 slots) per GPC, 8 GPCs
        const int kbp = (k_blocks + s - 1) / s;
        const int se = (k_blocks + kbp - 1) / kbp;
        if (se != s) continue;
        const long ctas = (long)n_tiles * se;
        const long waves = (ctas + slots - 1) / slots;
        const double cost = (double)waves * (kbp + 4.0) + (se > 1 ? 2.0 : 0.0);
        if (cost < best - 1e-9) {
            best = cost;
            best_s = se;
        }
    }
    if (forced > 0) best_s = forced < smax ? forced : smax;
    int kbp = (k_blocks + best_s - 1) / best_s;
    *kb_per_split = kbp;
    *nsplit = (k_blocks + kbp - 1) / kbp;
}
// Counters at the head of the GEMM workspace, partials after them. [0, 16384): the persistent kernel's split-K counters (int
// [0, 2048) tile arrivals, [2048, 4096) departures); [16384, 24576): the plain kernel's tile arrivals (l2_merge). Apart, because
// a decode program runs plain GEMMs (INT8G, INT4 g64 / g32) next to persistent-kernel ops on the same workspace.
constexpr size_t kGemmTileSemOffset = 16384;
constexpr size_t kGemmSemBytes = kGemmTileSemOffset + 2048 * sizeof(unsigned);

// partial slots of the plain kernel's split-K plan at this batch pad: [n_tiles][nsplit][bpad * 128] fp32, none unsplit
size_t gemm_partial_bytes(int n_tiles, int k_blocks, int bpad) {
    int nsplit, kbp;
    gemm_split(n_tiles, k_blocks, &nsplit, &kbp);
    return nsplit > 1 ? (size_t)n_tiles * nsplit * bpad * kGemmTileN * sizeof(float) : 0;
}

// Split-K plan of the persistent kernel: the n_tiles*k_blocks work list is cut into runs of `per` k-blocks, one per CTA.
// The run length is the smallest divisor of k_blocks that still gives every CTA at most one run (or whole tiles when there
// are more tiles than CTAs), so every CTA owns exactly one segment and the S = k_blocks / per contributors of a tile
// (S a power of two, at most 16, their partials within ws_partial_bytes) merge their partials together.
int sk_plan(int n_tiles, int k_blocks, int grid, int bpad, size_t ws_partial_bytes) {
    const long total = (long)n_tiles * k_blocks;
    const size_t slot = (size_t)bpad * kGemmTileN * sizeof(float);
    const int want = (int)((total + grid - 1) / grid);
    if (want >= k_blocks) return (want + k_blocks - 1) / k_blocks * k_blocks;   // whole tiles, possibly several per CTA
    for (int d = want; d <= k_blocks; ++d) {
        const int S = k_blocks / d;
        if (k_blocks % d == 0 && (S & (S - 1)) == 0 && S <= 16 && (size_t)n_tiles * S * slot <= ws_partial_bytes) return d;
    }
    return k_blocks;
}
// partial slots the plan needs at this grid and batch pad; a call with a smaller grid or batch pad picks a run at least as
// long, so it needs no more and gets the same plan from a workspace of this size
size_t sk_ws_bytes(int n_tiles, int k_blocks, int grid, int bpad) {
    const int per = sk_plan(n_tiles, k_blocks, grid, bpad, (size_t)-1);
    return per < k_blocks ? (size_t)n_tiles * (k_blocks / per) * bpad * kGemmTileN * sizeof(float) : 0;
}

// ---- peer regions
// A rank's peer-visible region: [2 parities][2 areas (one-shot / reduce-scatter, all-gather)][W sources][LL slot = 2 x message],
// then the per-CTA epochs at 2 * parity.
struct PeerStrides {
    size_t src, area, parity;
};
PeerStrides peer_strides(size_t max_message_bytes) {
    const size_t src = 2 * round_up(max_message_bytes, 256);   // LL doubles the bytes
    return {src, (size_t)kArMaxWorld * src, 2 * (size_t)kArMaxWorld * src};
}

bool valid_peer_group(int rank, int world) { return world >= 2 && world <= kArMaxWorld && rank >= 0 && rank < world; }

// The region pointers, epoch and strides of a peer kernel's parameters (PeerArParams and the GEMM's RsPush share the names).
template <typename P>
int set_peers(P& p, const char* who, void* const* regions, size_t max_message_bytes, int rank, int world) {
    const PeerStrides s = peer_strides(max_message_bytes);
    for (int r = 0; r < world; ++r) {
        ARG_CHECK(regions[r], "%s: region %d is null", who, r);
        p.region[r] = reinterpret_cast<uint8_t*>(regions[r]);
    }
    p.epoch = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(regions[rank]) + 2 * s.parity);
    p.src_stride = s.src;
    p.parity_stride = s.parity;
    p.rank = rank;
    p.world = world;
    return B200_OK;
}
int fill_ar_params(PeerArParams& p, void* const* regions, size_t max_message_bytes, int rank, int world) {
    p.area_stride = peer_strides(max_message_bytes).area;
    return set_peers(p, "peer collective", regions, max_message_bytes, rank, world);
}

}  // namespace

// ------------------------------------------------------------------------------------------------ decode program recorder
// A program is recorded from ordinary op calls, like a CUDA-graph capture (the reference captures its decode step with
// cudaStreamBeginCapture in cpp/cuda_graph/cuda_graph_runner.cc): between b200_program_begin and b200_program_end the
// calling thread's op calls are appended to the program instead of being launched. Consecutive ops the persistent kernel
// implements (weight-only GEMMs, norms, rope + append, embedding, block-table conversion) become ONE launch; every other
// op's launch (attention, FP16 GEMMs, argmax, all-reduce) is kept with its arguments and issued as its own launch in between.
struct b200_program {
    struct Item {
        bool segment = false;
        int first = 0, count = 0;          // ops[first, first+count)
        int bf16 = -1, bpad = -1, qfmt = -1;
        const char* name = nullptr;        // non-segment: the kernel and its recorded launch on a given stream
        std::function<cudaError_t(cudaStream_t)> issue;
    };
    std::vector<ProgOp> ops;
    std::vector<Item> items;
    ProgOp* d_ops = nullptr;
    unsigned* d_bar = nullptr;
    unsigned long long* trace = nullptr;
    bool finalized = false;
};

thread_local b200_program* b200_host::g_rec = nullptr;

int b200_host::record_launch(const char* name, std::function<cudaError_t(cudaStream_t)> issue) {
    b200_program::Item it;
    it.name = name;
    it.issue = std::move(issue);
    g_rec->items.push_back(std::move(it));
    return B200_OK;
}

namespace {

int rec_segment_op(const ProgOp& op, int bf16, int bpad, int qfmt) {
    b200_program* P = g_rec;
    auto compat = [](int a, int b) { return a < 0 || b < 0 || a == b; };
    if (!P->items.empty()) {
        b200_program::Item& it = P->items.back();
        if (it.segment && compat(it.bf16, bf16) && compat(it.bpad, bpad) && compat(it.qfmt, qfmt)) {
            if (it.bf16 < 0) it.bf16 = bf16;
            if (it.bpad < 0) it.bpad = bpad;
            if (it.qfmt < 0) it.qfmt = qfmt;
            P->ops.push_back(op);
            ++it.count;
            return B200_OK;
        }
    }
    b200_program::Item it;
    it.segment = true;
    it.first = (int)P->ops.size();
    it.count = 1;
    it.bf16 = bf16;
    it.bpad = bpad;
    it.qfmt = qfmt;
    P->ops.push_back(op);
    P->items.push_back(std::move(it));
    return B200_OK;
}
}  // namespace

extern "C" {

const char* b200_last_error(void) { return g_err.c_str(); }

int b200_set_pdl(int enable) {
    g_pdl.store(enable ? 1 : 0);
    return B200_OK;
}

uint64_t b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int b200_device_check(int device) {
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return fail(B200_EUNSUPPORTED, "no CUDA device %d: %s", device, cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return fail(B200_EUNSUPPORTED, "device %d is sm_%d%d, this library is sm_90a only", device, prop.major, prop.minor);
    if (!encode_fn()) return fail(B200_EUNSUPPORTED, "driver lacks cuTensorMapEncodeTiled");
    return B200_OK;
}

// ------------------------------------------------------------------------------------------------ launch-shape introspection
int b200_plan_attn_split(int units, int max_seq_len, int* nsplit, int* tiles_per_split) {
    ARG_CHECK(units > 0 && max_seq_len > 0 && nsplit && tiles_per_split, "plan_attn_split: bad argument");
    attn_split(units, (max_seq_len + kAttnTile - 1) / kAttnTile, nsplit, tiles_per_split);
    return B200_OK;
}

int b200_plan_gemm_split(int K, int N, int* nsplit, int* k_blocks_per_split) {
    ARG_CHECK(K > 0 && K % kGemmBK == 0 && N > 0 && nsplit && k_blocks_per_split, "plan_gemm_split: bad argument");
    gemm_split((N + kGemmTileN - 1) / kGemmTileN, K / kGemmBK, nsplit, k_blocks_per_split);
    return B200_OK;
}

// ------------------------------------------------------------------------------------------------ indexing
int b200_convert_block_table(int32_t* page_list, const int32_t* block_ids, int batch, int max_blocks, void* stream) {
    ARG_CHECK(page_list && block_ids, "convert_block_table: null pointer");
    ARG_CHECK(batch >= 0 && max_blocks >= 0, "convert_block_table: negative size");
    if (batch == 0 || max_blocks == 0) return B200_OK;
    if (g_rec) {
        ProgOp op{};
        op.type = kOpBlockTable;
        op.t.page_list = page_list;
        op.t.block_ids = block_ids;
        op.t.batch = batch;
        op.t.max_blocks = max_blocks;
        return rec_segment_op(op, -1, -1, -1);
    }
    const int total = batch * max_blocks;
    const int threads = 256, blocks = (total + threads - 1) / threads;
    return launch_or_record("convert_block_table_kernel", stream, [=](cudaStream_t s) {
        convert_block_table_kernel<<<blocks < 1024 ? blocks : 1024, threads, 0, s>>>(page_list, block_ids, batch, max_blocks);
        return cudaGetLastError();
    });
}

int b200_paged_attn_plan(const int32_t* input_lengths, const int32_t* sequence_lengths, const int32_t* prefix_lengths,
                         const int32_t* block_ids, int batch, int max_blocks, int tokens_per_block,
                         int32_t* paged_kv_last_page_len, int32_t* decode_page_indptr, int32_t* page_indice,
                         int32_t* batch_indice, int32_t* positions, void* stream) {
    if (batch == 0) return B200_OK;
    ARG_CHECK(batch > 0 && batch <= 1024, "paged_attn_plan: batch %d exceeds the single-CTA limit 1024", batch);
    ARG_CHECK(prefix_lengths || sequence_lengths, "paged_attn_plan: need either prefix_lengths or sequence_lengths");
    ARG_CHECK(!prefix_lengths || input_lengths, "paged_attn_plan: prefill mode needs input_lengths");
    ARG_CHECK(tokens_per_block > 0, "paged_attn_plan: tokens_per_block must be positive");
    ARG_CHECK(paged_kv_last_page_len && decode_page_indptr && batch_indice && positions, "paged_attn_plan: null output");
    ARG_CHECK(!block_ids || page_indice, "paged_attn_plan: block_ids given but page_indice is null");
    const int threads = (batch + 31) / 32 * 32;
    return launch_or_record("paged_attn_plan_kernel", stream, [=](cudaStream_t s) {
        paged_attn_plan_kernel<<<1, threads, 0, s>>>(input_lengths, sequence_lengths, prefix_lengths, block_ids, batch, max_blocks,
                                                     tokens_per_block, paged_kv_last_page_len, decode_page_indptr, page_indice,
                                                     batch_indice, positions);
        return cudaGetLastError();
    });
}

// ------------------------------------------------------------------------------------------------ attention
size_t b200_paged_decode_attn_workspace_bytes(size_t batch, size_t head_num, size_t kv_head_num, size_t max_seq_len) {
    size_t tiles = (max_seq_len + kAttnTile - 1) / kAttnTile;
    size_t ns = tiles < (size_t)kAttnMaxSplit ? (tiles ? tiles : 1) : (size_t)kAttnMaxSplit;
    // sized for one query row per sequence and the largest head_dim (256)
    const AttnWorkspace w = attn_workspace(batch, head_num, kv_head_num, 1, ns, 256);
    return w.sem + w.ml + w.o;
}

// beam_width > 0: the beam instance. `batch` then counts requests, each with beam_width sequences (rows of q, out, page_list and
// sequence_lengths), and shared_lengths [batch] says how much of a request's K/V its beams share; q_len is 1.
// tree_parents != null: the tree instance, parents [batch][q_len] of each sequence's q_len new tokens.
static int attn_impl(const void* q, const void* qkv, float rope_base, int q_len, int is_bf16, void* out, size_t head_num, size_t kv_head_num,
                     size_t head_dim, size_t batch, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size, const void* kv_pool,
                     const int32_t* page_list, const uint32_t* sequence_lengths, float q_scale, void* workspace, size_t workspace_bytes,
                     void* stream, int beam_width = 0, const int32_t* shared_lengths = nullptr, const int32_t* tree_parents = nullptr) {
    if (batch == 0) return B200_OK;
    ARG_CHECK((q || qkv) && out && kv_pool && page_list && sequence_lengths, "paged_decode_attn: null pointer");
    ARG_CHECK(head_dim == 64 || head_dim == 128 || head_dim == 256, "paged_decode_attn: head_dim %zu unsupported (64 / 128 / 256)", head_dim);
    ARG_CHECK(!qkv || head_dim == 128, "paged_decode_attn_rope: the fused rope is built for head_dim 128 (got %zu)", head_dim);
    ARG_CHECK(kv_head_num > 0 && head_num % kv_head_num == 0, "paged_decode_attn: head_num %zu not a multiple of kv_head_num %zu",
              head_num, kv_head_num);
    const int group = (int)(head_num / kv_head_num);
    // the fused rope loads q into one 16-row tile; the plain q load takes up to four
    ARG_CHECK(!qkv || group <= 16, "paged_decode_attn_rope: group size %d unsupported (1..16)", group);
    ARG_CHECK(group >= 1 && group <= kAttnMaxRows, "paged_decode_attn: group size %d unsupported (1..%d)", group, kAttnMaxRows);
    ARG_CHECK(group * q_len <= kAttnMaxRows, "paged_decode_attn: group %d x q_len %d exceeds the limit of %d query rows per (sequence, kv head)",
              group, q_len, kAttnMaxRows);
    ARG_CHECK(group * beam_width <= kAttnMaxRows,
              "paged_decode_attn_beam: group %d x beam_width %d exceeds the limit of %d query rows per (request, kv head)", group,
              beam_width, kAttnMaxRows);
    ARG_CHECK(page_size == 16 || page_size == 32 || page_size == 64 || page_size == 128,
              "paged_decode_attn: page_size %zu unsupported (16/32/64/128)", page_size);
    ARG_CHECK(max_seq_len >= 1, "paged_decode_attn: max_seq_len must be >= 1");
    ARG_CHECK(max_seq_len <= max_blocks_per_seq * page_size, "paged_decode_attn: max_seq_len %zu exceeds page table capacity %zu",
              max_seq_len, max_blocks_per_seq * page_size);
    ARG_CHECK(batch * kv_head_num <= 65535, "paged_decode_attn: batch*kv_heads %zu exceeds grid limit", batch * kv_head_num);
    ARG_CHECK(((uintptr_t)kv_pool & 15) == 0 && (((uintptr_t)q | (uintptr_t)qkv) & 3) == 0, "paged_decode_attn: misaligned pointer");

    const int slots = beam_width ? beam_width : q_len;   // query tokens or beams that share a CTA
    AttnBeamParams p{};
    p.beam_width = beam_width;
    p.shared_lens = shared_lengths;
    p.q = q;
    p.qkv = qkv;
    p.kv_pool_rw = const_cast<void*>(kv_pool);
    p.log2_base = qkv ? std::log2(rope_base) : 0.f;
    p.out = out;
    p.page_list = page_list;
    p.seq_lens = reinterpret_cast<const int32_t*>(sequence_lengths);
    p.B = (int)batch;
    p.Hq = (int)head_num;
    p.Hkv = (int)kv_head_num;
    p.group = group;
    p.q_len = q_len;
    p.M = (int)max_blocks_per_seq;
    p.T = (int)page_size;
    p.log2T = page_size == 16 ? 4 : page_size == 32 ? 5 : page_size == 64 ? 6 : 7;
    p.box_h = page_size < (size_t)kAttnTile ? (int)page_size : kAttnTile;
    p.boxes_per_tile = kAttnTile / p.box_h;
    p.scale_log2 = q_scale / std::sqrt((float)head_dim) * 1.4426950408889634f;
    const int max_tiles = (int)((max_seq_len + kAttnTile - 1) / kAttnTile);
    attn_split((int)(batch * kv_head_num), max_tiles, &p.nsplit, &p.tiles_per_split, (int)head_dim);

    if (p.nsplit > 8) {
        const AttnWorkspace w = attn_workspace(batch, head_num, kv_head_num, slots, p.nsplit, head_dim);
        ARG_CHECK(workspace && workspace_bytes >= w.sem + w.ml + w.o,
                  "paged_decode_attn: workspace too small (%zu < %zu)", workspace_bytes, w.sem + w.ml + w.o);
        p.sem = reinterpret_cast<int*>(workspace);
        p.ws_ml = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + w.sem);
        p.ws_o = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + w.sem + w.ml);
    }

    CUtensorMap map;
    {
        const cuuint64_t dims[4] = {(cuuint64_t)head_dim, (cuuint64_t)page_size, (cuuint64_t)kv_head_num, (cuuint64_t)1 << 31};
        const cuuint64_t strides[3] = {(cuuint64_t)head_dim * 2, (cuuint64_t)page_size * head_dim * 2,
                                       (cuuint64_t)kv_head_num * page_size * head_dim * 2};
        const cuuint32_t box[4] = {64, (cuuint32_t)p.box_h, 1, 1};
        int rc = make_map(&map, is_bf16 != 0, 4, kv_pool, dims, strides, box);
        if (rc) return rc;
    }
    const dim3 grid(p.nsplit, (unsigned)(batch * kv_head_num), 1);
    p.cluster_merge = (p.nsplit >= 2 && p.nsplit <= 8) ? 1 : 0;   // 2..8 splits merge in a cluster, more through the workspace
    const dim3 cluster(p.cluster_merge ? p.nsplit : 1);
    auto launch = [&](auto t, auto hd, auto rt, auto beam, auto tree) {
        constexpr auto kern = paged_decode_attn_kernel<decltype(t), decltype(hd)::value, decltype(rt)::value, decltype(beam)::value,
                                                       decltype(tree)::value>;
        const int smem = attn_smem_bytes(decltype(hd)::value);
        int rc = configure_once<kern>(smem);
        if (rc) return rc;
        if constexpr (decltype(tree)::value) {
            AttnTreeParams pt{};
            static_cast<AttnParams&>(pt) = p;
            pt.tree_parents = tree_parents;
            return launch_or_record("paged_decode_attn_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
                return launch_ex(kern, {grid, dim3(kAttnThreads), (size_t)smem, s, pdl, cluster}, map, pt);
            });
        } else {
            // (launch_ex converts p to the kernel's parameter type: the plain instances take its AttnParams part)
            return launch_or_record("paged_decode_attn_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
                return launch_ex(kern, {grid, dim3(kAttnThreads), (size_t)smem, s, pdl, cluster}, map, p);
            });
        }
    };
    // query rows in 16-row tiles: 1, 2 or 4 per (sequence or request, kv head)
    const int rows = group * slots;
    auto by_rows = [&](auto t, auto hd) {
        auto by_beam = [&](auto rt) {
            if (beam_width) return launch(t, hd, rt, std::true_type(), std::false_type());
            if (tree_parents) return launch(t, hd, rt, std::false_type(), std::true_type());
            return launch(t, hd, rt, std::false_type(), std::false_type());
        };
        if (rows <= 16) return by_beam(std::integral_constant<int, 1>());
        if (rows <= 32) return by_beam(std::integral_constant<int, 2>());
        return by_beam(std::integral_constant<int, 4>());
    };
    return by_dtype(is_bf16, [&](auto t) {
        if (head_dim == 64) return by_rows(t, std::integral_constant<int, 64>());
        if (head_dim == 128) return by_rows(t, std::integral_constant<int, 128>());
        return by_rows(t, std::integral_constant<int, 256>());
    });
}

int b200_paged_decode_attn(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                           size_t batch, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                           const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                           float q_scale, void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(q || batch == 0, "paged_decode_attn: null pointer");
    return attn_impl(q, nullptr, 0.f, 1, is_bf16, out, head_num, kv_head_num, head_dim, batch, max_blocks_per_seq, max_seq_len, page_size,
                     kv_pool, page_list, sequence_lengths, q_scale, workspace, workspace_bytes, stream);
}

int b200_paged_decode_attn_multi(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                 size_t batch, size_t q_len, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                 const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths, float q_scale,
                                 void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(q || batch == 0, "paged_decode_attn_multi: null pointer");
    ARG_CHECK(q_len >= 1 && q_len <= (size_t)kAttnMaxRows, "paged_decode_attn_multi: q_len %zu unsupported (1..%d)", q_len, kAttnMaxRows);
    return attn_impl(q, nullptr, 0.f, (int)q_len, is_bf16, out, head_num, kv_head_num, head_dim, batch, max_blocks_per_seq, max_seq_len,
                     page_size, kv_pool, page_list, sequence_lengths, q_scale, workspace, workspace_bytes, stream);
}

int b200_paged_decode_attn_rope(const void* qkv, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t batch, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size, void* kv_pool,
                                const int32_t* page_list, const uint32_t* sequence_lengths, float q_scale, float rope_base,
                                void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(qkv || batch == 0, "paged_decode_attn_rope: null pointer");
    ARG_CHECK(rope_base > 1.f, "paged_decode_attn_rope: rope_base must be > 1");
    return attn_impl(nullptr, qkv, rope_base, 1, is_bf16, out, head_num, kv_head_num, head_dim, batch, max_blocks_per_seq, max_seq_len,
                     page_size, kv_pool, page_list, sequence_lengths, q_scale, workspace, workspace_bytes, stream);
}

int b200_paged_decode_attn_beam(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t requests, size_t beam_width, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                                const int32_t* shared_lengths, float q_scale, void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(beam_width >= 1 && beam_width <= (size_t)kAttnMaxRows, "paged_decode_attn_beam: beam_width %zu unsupported (1..%d)",
              beam_width, kAttnMaxRows);
    ARG_CHECK(requests * kv_head_num <= 65535, "paged_decode_attn_beam: requests*kv_heads %zu exceeds grid limit", requests * kv_head_num);
    ARG_CHECK((q && shared_lengths) || requests == 0, "paged_decode_attn_beam: null pointer (q or shared_lengths)");
    return attn_impl(q, nullptr, 0.f, 1, is_bf16, out, head_num, kv_head_num, head_dim, requests, max_blocks_per_seq, max_seq_len,
                     page_size, kv_pool, page_list, sequence_lengths, q_scale, workspace, workspace_bytes, stream, (int)beam_width,
                     shared_lengths);
}

int b200_paged_decode_attn_tree(const void* q, int is_bf16, void* out, size_t head_num, size_t kv_head_num, size_t head_dim,
                                size_t batch, size_t q_len, size_t max_blocks_per_seq, size_t max_seq_len, size_t page_size,
                                const void* kv_pool, const int32_t* page_list, const uint32_t* sequence_lengths,
                                const int32_t* tree_parents, float q_scale, void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK((q && tree_parents) || batch == 0, "paged_decode_attn_tree: null pointer (q or tree_parents)");
    ARG_CHECK(q_len >= 1 && q_len <= (size_t)kAttnMaxRows, "paged_decode_attn_tree: q_len %zu unsupported (1..%d)", q_len, kAttnMaxRows);
    return attn_impl(q, nullptr, 0.f, (int)q_len, is_bf16, out, head_num, kv_head_num, head_dim, batch, max_blocks_per_seq, max_seq_len,
                     page_size, kv_pool, page_list, sequence_lengths, q_scale, workspace, workspace_bytes, stream, 0, nullptr,
                     tree_parents);
}

// ------------------------------------------------------------------------------------------------ GEMM
size_t b200_wo_gemm_packed_bytes(int fmt, int K, int N) {
    if (K <= 0 || N <= 0 || K % kGemmBK) return 0;
    const size_t n_tiles = (N + kGemmTileN - 1) / kGemmTileN, kb = K / kGemmBK;
    if (fmt == B200_FMT_INT4 || fmt == B200_FMT_INT4_G64 || fmt == B200_FMT_INT4_G32) return n_tiles * kb * gemm_w_bytes(fmt);
    if (fmt == B200_FMT_INT8) return n_tiles * kb * kW8BlockBytes;
    if (fmt == B200_FMT_INT8G) return n_tiles * kb * kW8GBlockBytes;
    if (fmt != B200_FMT_F16) return 0;
    return (size_t)N * K * 2;
}

int b200_pack_w4(const uint8_t* q_packed, const void* scales, const void* zeros_x_scales, int K, int N, int group,
                 void* blob, void* stream) {
    ARG_CHECK(q_packed && scales && zeros_x_scales && blob, "pack_w4: null pointer");
    ARG_CHECK(group == 128 || group == 64 || group == 32, "pack_w4: group size %d unsupported (128, 64 or 32)", group);
    ARG_CHECK(K > 0 && K % kGemmBK == 0, "pack_w4: K=%d must be a positive multiple of 128", K);
    ARG_CHECK(N > 0 && N % 2 == 0, "pack_w4: N=%d must be positive and even", N);
    const int fmt = group == 128 ? B200_FMT_INT4 : (group == 64 ? B200_FMT_INT4_G64 : B200_FMT_INT4_G32);
    const size_t words = b200_wo_gemm_packed_bytes(fmt, K, N) / 4;
    const int threads = 256;
    const size_t blocks = (words + threads - 1) / threads;
    pack_w4_kernel<<<(unsigned)(blocks < 65535 ? blocks : 65535), threads, 0, (cudaStream_t)stream>>>(
        q_packed, reinterpret_cast<const uint16_t*>(scales), reinterpret_cast<const uint16_t*>(zeros_x_scales), K, N, group,
        reinterpret_cast<uint8_t*>(blob));
    return launched("pack_w4_kernel");
}

int b200_pack_w8(const int8_t* q, int K, int N, void* blob, void* stream) {
    ARG_CHECK(q && blob, "pack_w8: null pointer");
    ARG_CHECK(K > 0 && K % kGemmBK == 0, "pack_w8: K=%d must be a positive multiple of 128", K);
    ARG_CHECK(N > 0, "pack_w8: N must be positive");
    const size_t bytes = b200_wo_gemm_packed_bytes(B200_FMT_INT8, K, N);
    const int threads = 256;
    const size_t blocks = (bytes + threads - 1) / threads;
    pack_w8_kernel<<<(unsigned)(blocks < 65535 ? blocks : 65535), threads, 0, (cudaStream_t)stream>>>(
        q, K, N, reinterpret_cast<uint8_t*>(blob));
    return launched("pack_w8_kernel");
}

int b200_pack_w8g(const int8_t* q, const void* scales, const void* zeros_x_scales, int K, int N, int group, void* blob,
                  void* stream) {
    ARG_CHECK(q && scales && zeros_x_scales && blob, "pack_w8g: null pointer");
    ARG_CHECK(group == kGemmBK, "pack_w8g: group size %d unsupported (128 only)", group);
    ARG_CHECK(K > 0 && K % kGemmBK == 0, "pack_w8g: K=%d must be a positive multiple of 128", K);
    ARG_CHECK(N > 0, "pack_w8g: N must be positive");
    const size_t bytes = b200_wo_gemm_packed_bytes(B200_FMT_INT8G, K, N);
    const int threads = 256;
    const size_t blocks = (bytes + threads - 1) / threads;
    pack_w8g_kernel<<<(unsigned)(blocks < 65535 ? blocks : 65535), threads, 0, (cudaStream_t)stream>>>(
        q, reinterpret_cast<const uint16_t*>(scales), reinterpret_cast<const uint16_t*>(zeros_x_scales), K, N,
        reinterpret_cast<uint8_t*>(blob));
    return launched("pack_w8g_kernel");
}

size_t b200_wo_gemm_workspace_bytes(int max_batch, int N, int K) {
    if (max_batch <= 0 || N <= 0 || K <= 0 || K % kGemmBK) return 0;
    const int n_tiles = (N + kGemmTileN - 1) / kGemmTileN;
    // partials of the plain kernel's split-K plan (any batch <= max_batch has a batch pad no larger) and of the persistent
    // kernel's, sized for its largest grid (2 CTAs per SM); the two never run at once, so they share the room
    const size_t plain = gemm_partial_bytes(n_tiles, K / kGemmBK, gemm_bpad(max_batch));
    const size_t persistent = sk_ws_bytes(n_tiles, K / kGemmBK, 2 * num_sms(), gemm_bpad(max_batch));
    return kGemmSemBytes + (plain > persistent ? plain : persistent);
}

// rs: the reduce-scatter push of b200_wo_gemm_rs, or null
static int wo_gemm_impl(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* col_scale,
                        const void* bias, void* y, void* workspace, size_t workspace_bytes, int flags, const RsPush* rs,
                        void* stream) {
    if (B == 0) return B200_OK;
    ARG_CHECK(fmt == B200_FMT_F16 || fmt == B200_FMT_INT8 || fmt == B200_FMT_INT4 || fmt == B200_FMT_INT8G || fmt == B200_FMT_INT4_G64 ||
                  fmt == B200_FMT_INT4_G32,
              "wo_gemm: unknown weight format %d", fmt);
    ARG_CHECK(x && w && y, "wo_gemm: null pointer");
    ARG_CHECK(B > 0 && B <= 128, "wo_gemm: batch %d unsupported (1..128 per call)", B);
    ARG_CHECK(K > 0 && K % kGemmBK == 0, "wo_gemm: K=%d must be a positive multiple of 128", K);
    ARG_CHECK(N > 0, "wo_gemm: N must be positive");
    ARG_CHECK(fmt != B200_FMT_INT8 || col_scale, "wo_gemm: INT8 needs col_scale");
    ARG_CHECK((((uintptr_t)x | (uintptr_t)w | (uintptr_t)y) & 15) == 0, "wo_gemm: x / w / y must be 16-byte aligned");
    const int n_tiles = (N + kGemmTileN - 1) / kGemmTileN;
    ARG_CHECK(n_tiles <= 2032, "wo_gemm: N=%d too large", N);   // persistent kernel: arrivals [0, 2048), departures [2048, 2048 + n_tiles)
    const int bpad = gemm_bpad(B);
    const bool silu_mul = (flags & B200_GEMM_SILU_MUL) != 0;
    ARG_CHECK(!silu_mul || N % 128 == 0, "wo_gemm: SILU_MUL needs N %% 128 == 0 (gate/up interleaved per 128-feature tile)");
    const bool use_pdl = (flags & B200_GEMM_PDL) || g_pdl.load();

    CUtensorMap xmap;
    {
        const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)B};
        const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
        const cuuint32_t box[2] = {64, (cuuint32_t)bpad};
        int rc = make_map(&xmap, is_bf16 != 0, 2, x, dims, strides, box);
        if (rc) return rc;
    }

    // ---- weight-only INT8 / INT4 at decode batches inside a decode program: an op of the persistent kernel (uniform split-K
    // merged through L2). Every other GEMM, and every call outside a program, uses the one-kernel-per-GEMM path below, which
    // needs no grid-wide barrier.
    const bool seg_capable = (fmt == B200_FMT_INT8 || fmt == B200_FMT_INT4) && bpad <= 64;   // INT8G / INT4 g64, g32 / FP16: cluster kernel only
    if (g_rec && seg_capable && !rs) {
        ARG_CHECK(workspace && workspace_bytes >= kGemmSemBytes, "wo_gemm: workspace of at least %zu bytes required", kGemmSemBytes);
        int grid = 0;
        int rc = by_dtype(is_bf16, [&](auto t) { return segment_grid<decltype(t)>(bpad, fmt, &grid); });
        if (rc) return rc;
        ProgOp op{};
        op.xmap = xmap;
        op.type = kOpGemm;
        op.fmt = fmt;
        SkGemmParams& g = op.g;
        g.w_blob = reinterpret_cast<const uint8_t*>(w);
        g.col_scale = col_scale;
        g.bias = bias;
        g.y = y;
        g.B = B;
        g.N = N;
        g.K = K;
        g.k_blocks = K / kGemmBK;
        g.n_tiles = n_tiles;
        g.total_kb = n_tiles * g.k_blocks;
        g.per_cta = sk_plan(n_tiles, g.k_blocks, grid, bpad, workspace_bytes - kGemmSemBytes);
        g.sem = reinterpret_cast<int*>(workspace);
        g.ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + kGemmSemBytes);
        g.silu_mul = silu_mul ? 1 : 0;
        return rec_segment_op(op, is_bf16 ? 1 : 0, bpad, fmt);
    }

    // ---- one kernel per GEMM, split-K merged by the last split CTA of a tile (gemm_cluster.cu)
    GemmParams p{};
    p.w_blob = reinterpret_cast<const uint8_t*>(w);
    p.col_scale = col_scale;
    p.bias = bias;
    p.y = y;
    p.B = B;
    p.N = N;
    p.K = K;
    p.k_blocks = K / kGemmBK;
    p.use_pdl = use_pdl ? 1 : 0;
    p.silu_mul = silu_mul ? 1 : 0;
    gemm_split(n_tiles, p.k_blocks, &p.nsplit, &p.kb_per_split);
    if (p.nsplit > 1 && !rs) {   // split-K partials merge through the workspace (l2_merge)
        const size_t need = kGemmSemBytes + gemm_partial_bytes(n_tiles, p.k_blocks, bpad);
        ARG_CHECK(workspace && workspace_bytes >= need,
                  "wo_gemm: workspace of %zu bytes too small for %d split-K partials of %d x %d (%zu bytes needed; size it "
                  "with b200_wo_gemm_workspace_bytes)", workspace ? workspace_bytes : (size_t)0, p.nsplit, B, N, need);
        p.tile_sem = reinterpret_cast<unsigned*>(reinterpret_cast<uint8_t*>(workspace) + kGemmTileSemOffset);
        p.ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + kGemmSemBytes);
    }
    CUtensorMap wmap;
    if (fmt == B200_FMT_F16) {
        const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
        const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
        const cuuint32_t box[2] = {64, (cuuint32_t)kGemmTileN};
        int rc = make_map(&wmap, is_bf16 != 0, 2, w, dims, strides, box);
        if (rc) return rc;
    } else {
        wmap = xmap;  // unused by the kernel
    }
    if (rs) {
        GemmParamsRs prs{};
        static_cast<GemmParams&>(prs) = p;
        prs.rs = *rs;
        return launch_cluster_gemm_rs(fmt, is_bf16 != 0, bpad, xmap, wmap, prs, n_tiles, (cudaStream_t)stream);
    }
    return launch_cluster_gemm(fmt, is_bf16 != 0, bpad, xmap, wmap, p, n_tiles, (cudaStream_t)stream);
}

int b200_wo_gemm(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* col_scale,
                 const void* bias, void* y, void* workspace, size_t workspace_bytes, int flags, void* stream) {
    return wo_gemm_impl(fmt, is_bf16, x, B, K, N, w, col_scale, bias, y, workspace, workspace_bytes, flags, nullptr, stream);
}

int b200_wo_gemm_rs(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* col_scale,
                    const void* bias, void* y, void* workspace, size_t workspace_bytes, int flags, void* const* regions,
                    size_t max_message_bytes, int rank, int world, void* stream) {
    ARG_CHECK(regions, "wo_gemm_rs: null regions");
    ARG_CHECK(fmt != B200_FMT_INT4_G64 && fmt != B200_FMT_INT4_G32, "wo_gemm_rs: INT4 group-64 / group-32 weights (format %d) unsupported", fmt);
    ARG_CHECK(valid_peer_group(rank, world), "wo_gemm_rs: bad rank/world %d/%d", rank, world);
    ARG_CHECK(N % 128 == 0 && N % (8 * world) == 0 && N <= 8192, "wo_gemm_rs: N=%d must be a multiple of 128 and of 8*world, <= 8192", N);
    ARG_CHECK((size_t)B * N * 2 <= max_message_bytes, "wo_gemm_rs: message of %zu bytes exceeds the region", (size_t)B * N * 2);
    ARG_CHECK(!(flags & B200_GEMM_SILU_MUL), "wo_gemm_rs: SILU_MUL cannot be combined with the reduce-scatter push");
    RsPush rs{};
    int rc = set_peers(rs, "wo_gemm_rs", regions, max_message_bytes, rank, world);
    if (rc) return rc;
    return wo_gemm_impl(fmt, is_bf16, x, B, K, N, w, col_scale, bias, y, workspace, workspace_bytes, flags, &rs, stream);
}

// ------------------------------------------------------------------------------------------------ glue ops
static constexpr int kNormMaxHidden = 12288;   // the stand-alone norm stages its row in shared memory: 48 KB at the limit

int b200_add_rmsnorm(const void* x, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                     float eps, void* stream) {
    if (rows == 0) return B200_OK;
    ARG_CHECK(x && gamma && y, "add_rmsnorm: null pointer");
    ARG_CHECK(hidden > 0 && hidden % 8 == 0 && hidden <= kNormMaxHidden, "add_rmsnorm: hidden=%d must be a multiple of 8, <= %d", hidden,
              kNormMaxHidden);
    if (g_rec && hidden <= kSegNormMaxHidden) {
        ProgOp op{};
        op.type = kOpNorm;
        op.n.x = x;
        op.n.residual = residual;
        op.n.gamma = gamma;
        op.n.y = y;
        op.n.rows = rows;
        op.n.hidden = hidden;
        op.n.eps = eps;
        return rec_segment_op(op, is_bf16 ? 1 : 0, -1, -1);
    }
    const int threads = hidden / 8 >= 512 ? 512 : (hidden / 8 >= 256 ? 256 : 128);
    const size_t smem = (size_t)hidden * sizeof(float);
    return by_dtype(is_bf16, [&](auto t) {
        using T = decltype(t);
        // the staged row is 48 KB at the limit: with the kernel's static s_red that is past the default dynamic limit
        const int rc = configure_once<add_rmsnorm_kernel<T>>(kNormMaxHidden * (int)sizeof(float));
        if (rc) return rc;
        return launch_or_record("add_rmsnorm_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(add_rmsnorm_kernel<T>, {dim3(rows), dim3(threads), smem, s, pdl}, (const T*)x, (T*)residual,
                             (const T*)gamma, (T*)y, hidden, eps);
        });
    });
}

int b200_qk_rmsnorm(void* qkv, const void* q_gamma, const void* k_gamma, const void* q_bias, const void* k_bias, int is_bf16,
                    int rows, int head_num, int kv_head_num, int head_dim, float eps, void* stream) {
    if (rows == 0) return B200_OK;
    ARG_CHECK(qkv && q_gamma && k_gamma, "qk_rmsnorm: null pointer");
    ARG_CHECK((q_bias == nullptr) == (k_bias == nullptr), "qk_rmsnorm: give both biases or none");
    ARG_CHECK(head_dim > 0 && head_dim % 64 == 0, "qk_rmsnorm: head_dim %d must be a multiple of 64 (fused_qk_rmsnorm.cu:104-106)", head_dim);
    ARG_CHECK(rows > 0 && head_num > 0 && kv_head_num > 0, "qk_rmsnorm: bad shape");
    const int units = rows * (head_num + kv_head_num), wpb = 8;
    const dim3 grid((units + wpb - 1) / wpb);
    return by_dtype(is_bf16, [&](auto t) {
        using T = decltype(t);
        return launch_or_record("qk_rmsnorm_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(qk_rmsnorm_kernel<T>, {grid, dim3(wpb * 32), 0, s, pdl}, (T*)qkv, (const T*)q_gamma, (const T*)k_gamma,
                             (const T*)q_bias, (const T*)k_bias, rows, head_num, kv_head_num, head_dim, eps);
        });
    });
}

int b200_silu_and_mul(const void* gate_up, void* y, int is_bf16, int rows, int inter, void* stream) {
    if (rows == 0) return B200_OK;
    ARG_CHECK(gate_up && y, "silu_and_mul: null pointer");
    ARG_CHECK(inter > 0 && inter % 2 == 0, "silu_and_mul: inter=%d must be positive and even", inter);
    const size_t total = (size_t)rows * inter / 2;
    const int threads = 256;
    const size_t blocks = (total + threads - 1) / threads;
    const unsigned g = (unsigned)(blocks < 4 * num_sms() * 8 ? blocks : 4 * num_sms() * 8);
    return by_dtype(is_bf16, [&](auto t) {
        using T = decltype(t);
        return launch_or_record("silu_and_mul_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(silu_and_mul_kernel<T>, {dim3(g), dim3(threads), 0, s, pdl}, (const T*)gate_up, (T*)y, rows, inter);
        });
    });
}

// the staged row is K 16-bit values in shared memory: 128 KB at the limit
static constexpr int kPermuteMaxK = 65536;

int b200_permute_cols(const void* x, const int32_t* perm, void* y, int is_bf16, int rows, int K, void* stream) {
    (void)is_bf16;   // a bit copy of 16-bit values: the same kernel serves both dtypes
    if (rows == 0) return B200_OK;
    ARG_CHECK(x && perm && y, "permute_cols: null pointer");
    ARG_CHECK(x != y, "permute_cols: x and y must not be the same buffer (the gather cannot run in place)");
    ARG_CHECK(rows > 0, "permute_cols: rows=%d must be positive", rows);
    ARG_CHECK(K > 0 && K % 8 == 0 && K <= kPermuteMaxK, "permute_cols: K=%d must be a positive multiple of 8, <= %d", K, kPermuteMaxK);
    ARG_CHECK((((uintptr_t)x | (uintptr_t)y | (uintptr_t)perm) & 15) == 0, "permute_cols: x / perm / y must be 16-byte aligned");
    const int rc = configure_once<permute_cols_kernel>(kPermuteMaxK * 2);
    if (rc) return rc;
    const int threads = K / 8 >= 512 ? 512 : (K / 8 >= 256 ? 256 : 128);
    return launch_or_record("permute_cols_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(permute_cols_kernel, {dim3(rows), dim3(threads), (size_t)K * 2, s, pdl}, (const uint16_t*)x, perm,
                         (uint16_t*)y, K);
    });
}

// The one host path of the six rope + append entry points (rope_append_kernel). plain: the plain Base rope at rope_base (no
// position ids, table, bias or logn); else the whole rope contract of *cfg. qkn: QK-RMSNorm first with p.q_gamma / p.k_gamma.
// Inside a decode program the plain one-token rope without QK-norm is the persistent kernel's rope op; every other mode is its
// own launch there.
static int rope_append_impl(const char* what, RopeAppendParams p, bool plain, float rope_base, const b200_rope_config* cfg, bool qkn,
                            int is_bf16, int q_len, void* stream) {
    RopeParams& r = p.r;
    ARG_CHECK(q_len >= 1, "%s: q_len %d must be >= 1", what, q_len);
    if (qkn) {
        ARG_CHECK(p.q_gamma && p.k_gamma, "%s: null gamma", what);
        ARG_CHECK(r.head_dim % 64 == 0 && r.head_dim <= kQkNormMaxD, "%s: head_dim %d must be 64, 128 or 256", what, r.head_dim);
    }
    if (r.B == 0) return B200_OK;
    ARG_CHECK(r.qkv && r.q_out && r.kv_pool && r.page_list && r.seq_lens && (plain || cfg), "%s: null pointer", what);
    ARG_CHECK(r.head_dim > 0 && r.head_dim % 2 == 0 && r.head_dim <= 512, "%s: head_dim %d unsupported", what, r.head_dim);
    ARG_CHECK(r.B > 0 && q_len <= 65535 && (long)r.B * q_len <= 0x7fffffffL, "%s: bad shape batch %d x q_len %d", what, r.B, q_len);
    if (plain) {
        ARG_CHECK(rope_base > 1.f, "%s: rope_base must be > 1", what);
        r.log2_base = std::log2(rope_base);
    } else {
        ARG_CHECK(cfg->style == 0 || (cfg->style >= 1 && cfg->style <= 7 && cfg->style != 2), "%s: rope style %d unsupported (Glm2 is out of scope)", what, cfg->style);
        ARG_CHECK(cfg->dim > 0 && cfg->dim % 2 == 0 && cfg->dim <= r.head_dim, "%s: rotary dim %d must be even and <= head_dim", what, cfg->dim);
        ARG_CHECK(cfg->style == 0 || cfg->base > 1.f, "%s: rope base must be > 1", what);
        ARG_CHECK(!p.cos_sin_cache || p.cache_positions > 0, "%s: a cos/sin cache needs its number of positions", what);
        ARG_CHECK(!p.use_logn || cfg->max_pos > 1, "%s: logn attention needs max_pos > 1", what);
        p.cfg = {cfg->style, cfg->dim, cfg->base, cfg->scale, cfg->factor1, cfg->factor2, cfg->max_pos, cfg->extrapolation_factor, cfg->mscale};
    }
    if (g_rec && plain && q_len == 1 && !qkn) {   // the persistent kernel's rope op appends one token per sequence, unnormed
        ProgOp op{};
        op.type = kOpRope;
        op.r = r;
        return rec_segment_op(op, is_bf16 ? 1 : 0, -1, -1);
    }
    const dim3 grid(r.B, r.head_num + 2 * r.kv_head_num, q_len), block(r.head_dim / 2);
    return by_dtype(is_bf16, [&](auto t) {
        using T = decltype(t);
        using Kernel = void (*)(RopeAppendParams);
        const Kernel kernels[2][2][2] = {   // [MULTI][QKN][PLAIN]
            {{rope_append_kernel<T, false, false, false>, rope_append_kernel<T, false, false, true>},
             {rope_append_kernel<T, false, true, false>, rope_append_kernel<T, false, true, true>}},
            {{rope_append_kernel<T, true, false, false>, rope_append_kernel<T, true, false, true>},
             {rope_append_kernel<T, true, true, false>, rope_append_kernel<T, true, true, true>}}};
        const Kernel kern = kernels[q_len > 1][qkn][plain];
        return launch_or_record("rope_append_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(kern, {grid, block, 0, s, pdl}, p);
        });
    });
}

int b200_rope_append(const void* qkv, void* q_out, void* kv_pool, const int32_t* page_list,
                     const int32_t* sequence_lengths, int is_bf16, int batch, int head_num, int kv_head_num,
                     int head_dim, int max_blocks_per_seq, int page_size, float rope_base, void* stream) {
    return b200_rope_append_multi(qkv, q_out, kv_pool, page_list, sequence_lengths, is_bf16, batch, head_num, kv_head_num, head_dim,
                                  max_blocks_per_seq, page_size, rope_base, 1, stream);
}

int b200_rope_append_multi(const void* qkv, void* q_out, void* kv_pool, const int32_t* page_list,
                           const int32_t* sequence_lengths, int is_bf16, int batch, int head_num, int kv_head_num,
                           int head_dim, int max_blocks_per_seq, int page_size, float rope_base, int q_len, void* stream) {
    const RopeAppendParams p{{qkv, q_out, kv_pool, page_list, sequence_lengths, batch, head_num, kv_head_num, head_dim, max_blocks_per_seq, page_size}};
    return rope_append_impl("rope_append", p, true, rope_base, nullptr, false, is_bf16, q_len, stream);
}

int b200_qk_norm_rope_append(const void* qkv, const void* q_gamma, const void* k_gamma, float eps, void* q_out, void* kv_pool,
                             const int32_t* page_list, const int32_t* sequence_lengths, int is_bf16, int batch, int head_num,
                             int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, float rope_base, int q_len,
                             void* stream) {
    RopeAppendParams p{{qkv, q_out, kv_pool, page_list, sequence_lengths, batch, head_num, kv_head_num, head_dim, max_blocks_per_seq, page_size}};
    p.q_gamma = q_gamma;
    p.k_gamma = k_gamma;
    p.eps = eps;
    return rope_append_impl("qk_norm_rope_append", p, true, rope_base, nullptr, true, is_bf16, q_len, stream);
}

int b200_rope_append_ex(const void* qkv, const void* qkv_bias, void* q_out, void* kv_pool, const int32_t* page_list,
                        const int32_t* sequence_lengths, const int32_t* position_ids, const float* cos_sin_cache,
                        int cache_positions, const b200_rope_config* cfg, int use_logn_attn, int is_bf16, int batch, int head_num,
                        int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, void* stream) {
    return b200_rope_append_ex_multi(qkv, qkv_bias, q_out, kv_pool, page_list, sequence_lengths, position_ids, cos_sin_cache,
                                     cache_positions, cfg, use_logn_attn, is_bf16, batch, head_num, kv_head_num, head_dim,
                                     max_blocks_per_seq, page_size, 1, stream);
}

int b200_rope_append_ex_multi(const void* qkv, const void* qkv_bias, void* q_out, void* kv_pool, const int32_t* page_list,
                              const int32_t* sequence_lengths, const int32_t* position_ids, const float* cos_sin_cache,
                              int cache_positions, const b200_rope_config* cfg, int use_logn_attn, int is_bf16, int batch,
                              int head_num, int kv_head_num, int head_dim, int max_blocks_per_seq, int page_size, int q_len,
                              void* stream) {
    const RopeAppendParams p{{qkv, q_out, kv_pool, page_list, sequence_lengths, batch, head_num, kv_head_num, head_dim, max_blocks_per_seq, page_size},
                             qkv_bias, position_ids, reinterpret_cast<const float2*>(cos_sin_cache), cache_positions, {}, use_logn_attn};
    return rope_append_impl("rope_append_ex", p, false, 0.f, cfg, false, is_bf16, q_len, stream);
}

int b200_qk_norm_rope_append_ex(const void* qkv, const void* q_gamma, const void* k_gamma, float eps, void* q_out, void* kv_pool,
                                const int32_t* page_list, const int32_t* sequence_lengths, const int32_t* position_ids,
                                const float* cos_sin_cache, int cache_positions, const b200_rope_config* cfg, int use_logn_attn,
                                int is_bf16, int batch, int head_num, int kv_head_num, int head_dim, int max_blocks_per_seq,
                                int page_size, int q_len, void* stream) {
    const RopeAppendParams p{{qkv, q_out, kv_pool, page_list, sequence_lengths, batch, head_num, kv_head_num, head_dim, max_blocks_per_seq, page_size},
                             nullptr, position_ids, reinterpret_cast<const float2*>(cos_sin_cache), cache_positions, {}, use_logn_attn,
                             q_gamma, k_gamma, eps};
    return rope_append_impl("qk_norm_rope_append_ex", p, false, 0.f, cfg, true, is_bf16, q_len, stream);
}

int b200_embedding(const int32_t* ids, const void* table, void* out, int is_bf16, int rows, int hidden, void* stream) {
    (void)is_bf16;
    if (rows == 0) return B200_OK;
    ARG_CHECK(ids && table && out, "embedding: null pointer");
    ARG_CHECK(hidden > 0 && hidden % 8 == 0, "embedding: hidden=%d must be a multiple of 8", hidden);
    if (g_rec) {
        ProgOp op{};
        op.type = kOpEmbed;
        op.e.ids = ids;
        op.e.table = table;
        op.e.out = out;
        op.e.rows = rows;
        op.e.hidden = hidden;
        return rec_segment_op(op, -1, -1, -1);
    }
    return launch_or_record("embedding_kernel", stream, [=](cudaStream_t s) {
        embedding_kernel<__half><<<rows, 128, 0, s>>>(ids, (const __half*)table, (__half*)out, hidden);
        return cudaGetLastError();
    });
}

int b200_argmax(const void* logits, int dtype, int rows, int vocab, int32_t* out, void* stream) {
    if (rows == 0) return B200_OK;
    ARG_CHECK(logits && out, "argmax: null pointer");
    ARG_CHECK(vocab > 0, "argmax: vocab must be positive");
    ARG_CHECK(dtype >= 0 && dtype <= 2, "argmax: dtype %d unknown (0 fp16, 1 bf16, 2 fp32)", dtype);
    auto launch = [&](auto t) {
        using T = decltype(t);
        return launch_or_record("argmax_kernel", stream, [=](cudaStream_t s) {
            argmax_kernel<T><<<rows, 1024, 0, s>>>((const T*)logits, vocab, out);
            return cudaGetLastError();
        });
    };
    return dtype == 2 ? launch(0.f) : by_dtype(dtype == 1, launch);
}

int b200_sample(float* logits, int rows, int vocab, const int32_t* history, const int32_t* hist_len, int hist_stride,
                int32_t* count_ws, const float* temperature, const float* repetition, const float* presence,
                const float* frequency, const int32_t* top_k, const float* top_p, const float* min_p, const float* uniform,
                const uint8_t* process, int32_t* token_out, float* token_prob_out, float* probs_out, void* stream) {
    if (rows == 0) return B200_OK;
    ARG_CHECK(logits && top_k && top_p && uniform && token_out, "sample: null pointer");
    ARG_CHECK(rows > 0 && rows <= 65535 && vocab > 0, "sample: bad shape [%d, %d]", rows, vocab);
    ARG_CHECK(!history || (hist_len && hist_stride > 0), "sample: history needs hist_len and a positive stride");
    ARG_CHECK(!(repetition || presence || frequency) || (history && count_ws), "sample: penalties need history and count_ws");
    SampleParams p{};
    p.logits = logits;
    p.probs_out = probs_out;
    p.history = history;
    p.hist_len = hist_len;
    p.count_ws = count_ws;
    p.temperature = temperature;
    p.repetition = repetition;
    p.presence = presence;
    p.frequency = frequency;
    p.top_k = top_k;
    p.top_p = top_p;
    p.min_p = min_p;
    p.uniform = uniform;
    p.process = process;
    p.token_out = token_out;
    p.token_prob_out = token_prob_out;
    p.rows = rows;
    p.vocab = vocab;
    p.hist_stride = hist_stride;
    return launch_or_record("sample_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(sample_kernel, {dim3(rows), dim3(kSampleThreads), 0, s, pdl}, p);
    });
}

int b200_spec_verify(const float* target_probs, const int32_t* target_ids, const float* draft_probs, const int32_t* draft_tokens,
                     const float* uniform, int batch, int num_draft, int vocab, int32_t* out_tokens, int32_t* accepted, void* stream) {
    ARG_CHECK(batch >= 0 && batch <= 65535, "spec_verify: batch %d unsupported (0..65535)", batch);
    ARG_CHECK(num_draft >= 0, "spec_verify: num_draft %d must be >= 0", num_draft);
    ARG_CHECK(vocab > 0, "spec_verify: vocab must be positive");
    if (batch == 0) return B200_OK;
    ARG_CHECK(out_tokens && accepted && (draft_tokens || num_draft == 0), "spec_verify: null pointer");
    ARG_CHECK(target_probs || target_ids, "spec_verify: need target_probs (sampling) or target_ids (greedy)");
    ARG_CHECK(!target_probs || uniform, "spec_verify: sampling mode needs uniform");
    ARG_CHECK(!draft_probs || target_probs, "spec_verify: draft_probs need target_probs");
    SpecVerifyParams p{};
    p.target_probs = target_probs;
    p.target_ids = target_ids;
    p.draft_probs = draft_probs;
    p.draft_tokens = draft_tokens;
    p.uniform = uniform;
    p.out_tokens = out_tokens;
    p.accepted = accepted;
    p.num_nodes = num_draft + 1;
    p.vocab = vocab;
    return launch_or_record("spec_verify_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(spec_verify_kernel, {dim3(batch), dim3(kSampleThreads), 0, s, pdl}, p);
    });
}

int b200_spec_verify_tree(const float* target_probs, const int32_t* target_ids, const int32_t* tree_parents, const int32_t* node_tokens,
                          const float* uniform, int batch, int n, int vocab, int32_t* out_tokens, int32_t* accepted,
                          int32_t* accepted_path, void* stream) {
    ARG_CHECK(batch >= 0 && batch <= 65535, "spec_verify_tree: batch %d unsupported (0..65535)", batch);
    ARG_CHECK(n >= 1 && n <= kSpecTreeMaxNodes, "spec_verify_tree: n %d unsupported (1..%d)", n, kSpecTreeMaxNodes);
    ARG_CHECK(vocab > 0, "spec_verify_tree: vocab must be positive");
    if (batch == 0) return B200_OK;
    ARG_CHECK(tree_parents && node_tokens && out_tokens && accepted && accepted_path, "spec_verify_tree: null pointer");
    ARG_CHECK(target_probs || target_ids, "spec_verify_tree: need target_probs (sampling) or target_ids (greedy)");
    ARG_CHECK(!target_probs || uniform, "spec_verify_tree: sampling mode needs uniform");
    SpecVerifyParams p{};
    p.target_probs = target_probs;
    p.target_ids = target_ids;
    p.draft_tokens = node_tokens;
    p.parents = tree_parents;
    p.uniform = uniform;
    p.out_tokens = out_tokens;
    p.accepted = accepted;
    p.accepted_path = accepted_path;
    p.num_nodes = n;
    p.vocab = vocab;
    return launch_or_record("spec_verify_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(spec_verify_kernel, {dim3(batch), dim3(kSampleThreads), 0, s, pdl}, p);
    });
}

int b200_kv_compact_path(void* const* kv_pools, int layers, int kv_head_num, int head_dim, int page_size, const int32_t* page_list,
                         int max_blocks_per_seq, const int32_t* sequence_lengths, const int32_t* accepted_path, const int32_t* accepted,
                         int batch, int n, void* stream) {
    ARG_CHECK(layers >= 1 && layers <= kCompactMaxLayers, "kv_compact_path: layers %d unsupported (1..%d)", layers, kCompactMaxLayers);
    ARG_CHECK(kv_head_num >= 1 && kv_head_num <= 65535, "kv_compact_path: kv_head_num %d unsupported (1..65535)", kv_head_num);
    ARG_CHECK(head_dim == 64 || head_dim == 128 || head_dim == 256, "kv_compact_path: head_dim %d unsupported (64 / 128 / 256)", head_dim);
    ARG_CHECK(page_size >= 1 && max_blocks_per_seq >= 1, "kv_compact_path: page_size and max_blocks_per_seq must be positive");
    ARG_CHECK((long long)page_size * max_blocks_per_seq <= 0x7fffffffLL, "kv_compact_path: page table capacity exceeds 2^31 - 1");
    ARG_CHECK(n >= 1 && n <= kSpecTreeMaxNodes, "kv_compact_path: n %d unsupported (1..%d)", n, kSpecTreeMaxNodes);
    ARG_CHECK(batch >= 0, "kv_compact_path: batch %d must be >= 0", batch);
    if (batch == 0) return B200_OK;
    ARG_CHECK(kv_pools && page_list && sequence_lengths && accepted_path && accepted, "kv_compact_path: null pointer");
    KvCompactParams p{};
    for (int l = 0; l < layers; ++l) {
        ARG_CHECK(kv_pools[l], "kv_compact_path: pool of layer %d is null", l);
        ARG_CHECK(((uintptr_t)kv_pools[l] & 15) == 0, "kv_compact_path: pool of layer %d is not 16-byte aligned", l);
        p.pools[l] = kv_pools[l];
    }
    p.page_list = page_list;
    p.seq_lens = sequence_lengths;
    p.path = accepted_path;
    p.accepted = accepted;
    p.kv_head_num = kv_head_num;
    p.head_dim = head_dim;
    p.page_size = page_size;
    p.max_blocks = max_blocks_per_seq;
    p.n = n;
    const dim3 grid(batch, kv_head_num, layers);
    return launch_or_record("kv_compact_path_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(kv_compact_path_kernel, {grid, dim3(head_dim / 4), 0, s, pdl}, p);
    });
}

namespace {
// Byte offsets of the beam step's workspace arrays (BeamParams), each 256-byte aligned; total = 0 for an unsupported shape.
struct BeamWorkspace {
    size_t count, chunk_stat, chunk_val, chunk_idx, row_stat, row_val, row_idx, total;
};
BeamWorkspace beam_workspace(int batch, int beam_width, int vocab) {
    BeamWorkspace w{};
    if (batch < 0 || beam_width < 1 || beam_width > kBeamMaxWidth || vocab < 2 * beam_width || vocab > (1 << 26)) return w;
    const size_t rows = (size_t)batch * beam_width, S = (vocab + kBeamChunk - 1) / kBeamChunk, K = 2 * beam_width;
    if (S * K > (size_t)kBeamMaxItems) return w;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o = round_up(o + bytes, 256);
        return at;
    };
    w.count = take((rows + batch) * 4);
    w.chunk_stat = take(rows * S * 8);
    w.chunk_val = take(rows * S * K * 4);
    w.chunk_idx = take(rows * S * K * 4);
    w.row_stat = take(rows * 8);
    w.row_val = take(rows * K * 4);
    w.row_idx = take(rows * K * 4);
    w.total = o;
    return w;
}
}  // namespace

size_t b200_beam_search_step_workspace_bytes(int batch, int beam_width, int vocab) {
    return beam_workspace(batch, beam_width, vocab).total;
}

int b200_beam_search_step(const void* logits, int dtype, const float* cum_log_probs, int batch, int beam_width, int vocab, int eos_id,
                          int32_t* cand_token, int32_t* cand_parent, float* cand_score, int32_t* next_token, int32_t* next_parent,
                          float* next_cum, void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(beam_width >= 1 && beam_width <= kBeamMaxWidth, "beam_search_step: beam_width %d unsupported (1..%d)", beam_width,
              kBeamMaxWidth);
    ARG_CHECK(vocab >= 2 * beam_width, "beam_search_step: vocab %d must be >= 2 * beam_width (%d)", vocab, 2 * beam_width);
    ARG_CHECK(vocab <= (1 << 26), "beam_search_step: vocab %d exceeds %d", vocab, 1 << 26);
    ARG_CHECK((size_t)(vocab + kBeamChunk - 1) / kBeamChunk * 2 * beam_width <= (size_t)kBeamMaxItems,
              "beam_search_step: vocab %d x beam_width %d exceeds the row merge (ceil(vocab / %d) * 2 * beam_width <= %d)", vocab,
              beam_width, kBeamChunk, kBeamMaxItems);
    ARG_CHECK(dtype >= 0 && dtype <= 2, "beam_search_step: dtype %d unknown (0 fp16, 1 bf16, 2 fp32)", dtype);
    ARG_CHECK(batch >= 0 && (long)batch * beam_width <= 65535, "beam_search_step: batch %d x beam_width %d exceeds 65535 rows", batch,
              beam_width);
    if (batch == 0) return B200_OK;
    ARG_CHECK(logits && cum_log_probs && cand_token && cand_parent && cand_score && next_token && next_parent && next_cum,
              "beam_search_step: null pointer");
    const BeamWorkspace w = beam_workspace(batch, beam_width, vocab);
    ARG_CHECK(workspace && workspace_bytes >= w.total,
              "beam_search_step: workspace too small (%zu < %zu bytes, see b200_beam_search_step_workspace_bytes)",
              workspace ? workspace_bytes : (size_t)0, w.total);
    char* ws = static_cast<char*>(workspace);
    BeamParams p{};
    p.logits = logits;
    p.cum = cum_log_probs;
    p.count = reinterpret_cast<uint32_t*>(ws + w.count);
    p.chunk_stat = reinterpret_cast<float2*>(ws + w.chunk_stat);
    p.chunk_val = reinterpret_cast<float*>(ws + w.chunk_val);
    p.chunk_idx = reinterpret_cast<uint32_t*>(ws + w.chunk_idx);
    p.row_stat = reinterpret_cast<float2*>(ws + w.row_stat);
    p.row_val = reinterpret_cast<float*>(ws + w.row_val);
    p.row_idx = reinterpret_cast<uint32_t*>(ws + w.row_idx);
    p.cand_token = cand_token;
    p.cand_parent = cand_parent;
    p.cand_score = cand_score;
    p.next_token = next_token;
    p.next_parent = next_parent;
    p.next_cum = next_cum;
    p.W = beam_width;
    p.V = vocab;
    p.S = (vocab + kBeamChunk - 1) / kBeamChunk;
    p.eos = eos_id;
    auto launch = [&](auto t) {
        return launch_or_record("beam_search_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(beam_search_kernel<decltype(t)>, {dim3(p.S, batch * beam_width), dim3(kBeamThreads), 0, s, pdl}, p);
        });
    };
    return dtype == 2 ? launch(0.f) : by_dtype(dtype == 1, launch);
}

size_t b200_beam_hypotheses_state_bytes(int batch, int beam_width, int max_len) {
    if (batch < 0 || beam_width < 1 || beam_width > kBeamMaxWidth || max_len < 1 || max_len > (1 << 24)) return 0;
    return (size_t)batch * beam_hyps_stride(beam_width, max_len);
}

// The checks both beam-hypothesis entries share
#define BEAM_HYPS_CHECKS(who)                                                                                                   \
    ARG_CHECK(beam_width >= 1 && beam_width <= kBeamMaxWidth, who ": beam_width %d unsupported (1..%d)", beam_width,          \
              kBeamMaxWidth);                                                                                                 \
    ARG_CHECK(max_len >= 1 && max_len <= (1 << 24), who ": max_len %d unsupported (1..%d)", max_len, 1 << 24);                \
    ARG_CHECK(batch >= 0 && batch <= 65535, who ": batch %d unsupported (0..65535)", batch);                                  \
    ARG_CHECK(hist_stride >= 1 && gen_start >= 0, who ": hist_stride %d must be >= 1 and gen_start %d >= 0", hist_stride,     \
              gen_start)

int b200_beam_hypotheses_update(const int32_t* cand_token, const int32_t* cand_parent, const float* cand_score, const int32_t* history,
                                const int32_t* hist_len, int hist_stride, int gen_start, int batch, int beam_width, int eos_id,
                                const float* length_penalty, const int32_t* early_stopping, int max_len, void* state,
                                size_t state_bytes, int32_t* done, void* stream) {
    BEAM_HYPS_CHECKS("beam_hypotheses_update");
    ARG_CHECK(eos_id >= 0, "beam_hypotheses_update: eos_id %d must be >= 0", eos_id);
    if (batch == 0) return B200_OK;
    ARG_CHECK(cand_token && cand_parent && cand_score && history && hist_len && length_penalty && early_stopping && state && done,
              "beam_hypotheses_update: null pointer");
    const size_t need = b200_beam_hypotheses_state_bytes(batch, beam_width, max_len);
    ARG_CHECK(state_bytes >= need, "beam_hypotheses_update: state too small (%zu < %zu bytes, see b200_beam_hypotheses_state_bytes)",
              state_bytes, need);
    BeamHypsParams p{};
    p.cand_token = cand_token;
    p.cand_parent = cand_parent;
    p.cand_score = cand_score;
    p.history = history;
    p.hist_len = hist_len;
    p.length_penalty = length_penalty;
    p.early_stopping = early_stopping;
    p.state = static_cast<char*>(state);
    p.done = done;
    p.W = beam_width;
    p.max_len = max_len;
    p.hist_stride = hist_stride;
    p.gen_start = gen_start;
    p.eos = eos_id;
    return launch_or_record("beam_hyps_update_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(beam_hyps_update_kernel, {dim3(batch), dim3(kBeamHypThreads), 0, s, pdl}, p);
    });
}

int b200_beam_hypotheses_finalize(const void* state, size_t state_bytes, const int32_t* done, const float* beam_cum,
                                  const int32_t* history, const int32_t* hist_len, int hist_stride, int gen_start, int batch,
                                  int beam_width, int n, int max_len, const float* length_penalty, int32_t* out_tokens,
                                  int32_t* out_len, float* out_score, float* out_cum, void* stream) {
    BEAM_HYPS_CHECKS("beam_hypotheses_finalize");
    ARG_CHECK(n >= 1 && n <= beam_width, "beam_hypotheses_finalize: n %d unsupported (1..beam_width %d)", n, beam_width);
    if (batch == 0) return B200_OK;
    ARG_CHECK(state && done && beam_cum && history && hist_len && length_penalty && out_tokens && out_len && out_score && out_cum,
              "beam_hypotheses_finalize: null pointer");
    const size_t need = b200_beam_hypotheses_state_bytes(batch, beam_width, max_len);
    ARG_CHECK(state_bytes >= need, "beam_hypotheses_finalize: state too small (%zu < %zu bytes, see b200_beam_hypotheses_state_bytes)",
              state_bytes, need);
    BeamHypsParams p{};
    p.beam_cum = beam_cum;
    p.history = history;
    p.hist_len = hist_len;
    p.length_penalty = length_penalty;
    p.state = const_cast<char*>(static_cast<const char*>(state));
    p.done = const_cast<int32_t*>(done);
    p.out_tokens = out_tokens;
    p.out_len = out_len;
    p.out_score = out_score;
    p.out_cum = out_cum;
    p.W = beam_width;
    p.n = n;
    p.max_len = max_len;
    p.hist_stride = hist_stride;
    p.gen_start = gen_start;
    return launch_or_record("beam_hyps_finalize_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
        return launch_ex(beam_hyps_finalize_kernel, {dim3(batch), dim3(kBeamHypThreads), 0, s, pdl}, p);
    });
}
#undef BEAM_HYPS_CHECKS

namespace {
// Byte offsets of the log-prob kernel's workspace arrays (LogprobParams), each 256-byte aligned; total = 0 for an unsupported
// shape.
struct LogprobWorkspace {
    size_t count, chunk_stat, chunk_val, chunk_idx, total;
};
LogprobWorkspace logprob_workspace(int rows, int vocab, int top_n) {
    LogprobWorkspace w{};
    const size_t S = vocab > 0 ? (vocab + kBeamChunk - 1) / kBeamChunk : 0;
    if (rows < 0 || rows > 65535 || vocab < 1 || vocab > (1 << 26) || top_n < 0 || top_n > kLogprobMaxTopN || top_n > vocab ||
        S * top_n > (size_t)kBeamMaxItems)
        return w;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o = round_up(o + bytes, 256);
        return at;
    };
    w.count = take((size_t)max(rows, 1) * 4);
    w.chunk_stat = take((size_t)rows * S * 8);
    w.chunk_val = take((size_t)rows * S * top_n * 4);
    w.chunk_idx = take((size_t)rows * S * top_n * 4);
    w.total = o;
    return w;
}
}  // namespace

size_t b200_token_logprobs_workspace_bytes(int rows, int vocab, int top_n) { return logprob_workspace(rows, vocab, top_n).total; }

int b200_token_logprobs(const void* logits, int dtype, int rows, int vocab, int top_n, const int32_t* tokens, float* token_logprob,
                        int32_t* top_ids, float* top_logprobs, void* workspace, size_t workspace_bytes, void* stream) {
    ARG_CHECK(rows >= 0 && rows <= 65535, "token_logprobs: rows %d unsupported (0..65535)", rows);
    ARG_CHECK(vocab > 0 && vocab <= (1 << 26), "token_logprobs: vocab %d unsupported (1..%d)", vocab, 1 << 26);
    ARG_CHECK(top_n >= 0 && top_n <= kLogprobMaxTopN && top_n <= vocab, "token_logprobs: top_n %d unsupported (0..min(%d, vocab))",
              top_n, kLogprobMaxTopN);
    ARG_CHECK((size_t)(vocab + kBeamChunk - 1) / kBeamChunk * top_n <= (size_t)kBeamMaxItems,
              "token_logprobs: vocab %d x top_n %d exceeds the row merge (ceil(vocab / %d) * top_n <= %d)", vocab, top_n, kBeamChunk,
              kBeamMaxItems);
    ARG_CHECK(dtype >= 0 && dtype <= 2, "token_logprobs: dtype %d unknown (0 fp16, 1 bf16, 2 fp32)", dtype);
    if (rows == 0) return B200_OK;
    ARG_CHECK(logits && (!tokens || token_logprob) && (top_n == 0 || (top_ids && top_logprobs)), "token_logprobs: null pointer");
    const LogprobWorkspace w = logprob_workspace(rows, vocab, top_n);
    ARG_CHECK(workspace && workspace_bytes >= w.total,
              "token_logprobs: workspace too small (%zu < %zu bytes, see b200_token_logprobs_workspace_bytes)",
              workspace ? workspace_bytes : (size_t)0, w.total);
    char* ws = static_cast<char*>(workspace);
    LogprobParams p{};
    p.logits = logits;
    p.tokens = tokens;
    p.token_logprob = token_logprob;
    p.top_ids = top_ids;
    p.top_logprobs = top_logprobs;
    p.count = reinterpret_cast<uint32_t*>(ws + w.count);
    p.chunk_stat = reinterpret_cast<float2*>(ws + w.chunk_stat);
    p.chunk_val = reinterpret_cast<float*>(ws + w.chunk_val);
    p.chunk_idx = reinterpret_cast<uint32_t*>(ws + w.chunk_idx);
    p.V = vocab;
    p.S = (vocab + kBeamChunk - 1) / kBeamChunk;
    p.top_n = top_n;
    auto launch = [&](auto t) {
        return launch_or_record("token_logprobs_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(token_logprobs_kernel<decltype(t)>, {dim3(p.S, rows), dim3(kBeamThreads), 0, s, pdl}, p);
        });
    };
    return dtype == 2 ? launch(0.f) : by_dtype(dtype == 1, launch);
}

int b200_ban_repeat_ngram(void* logits, int dtype, int rows, int vocab, const int32_t* history, const int32_t* hist_len, int hist_stride,
                          const int32_t* ngram_size, void* stream) {
    ARG_CHECK(rows >= 0 && rows <= 65535, "ban_repeat_ngram: rows %d unsupported (0..65535)", rows);
    ARG_CHECK(vocab > 0, "ban_repeat_ngram: vocab must be positive");
    ARG_CHECK(dtype >= 0 && dtype <= 2, "ban_repeat_ngram: dtype %d unknown (0 fp16, 1 bf16, 2 fp32)", dtype);
    ARG_CHECK(hist_stride > 0, "ban_repeat_ngram: hist_stride must be positive");
    if (rows == 0) return B200_OK;
    ARG_CHECK(logits && history && hist_len && ngram_size, "ban_repeat_ngram: null pointer");
    BanNgramParams p{};
    p.logits = logits;
    p.history = history;
    p.hist_len = hist_len;
    p.ngram_size = ngram_size;
    p.vocab = vocab;
    p.hist_stride = hist_stride;
    auto launch = [&](auto t) {
        return launch_or_record("ban_repeat_ngram_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(ban_repeat_ngram_kernel<decltype(t)>, {dim3(rows), dim3(256), 0, s, pdl}, p);
        });
    };
    return dtype == 2 ? launch(0.f) : by_dtype(dtype == 1, launch);
}

int b200_constrain_logits(void* logits, int dtype, int rows, int vocab, const int32_t* bitmask, int mask_stride,
                          const int32_t* bias_offsets, const int32_t* bias_ids, const float* bias_values, void* stream) {
    ARG_CHECK(rows >= 1 && rows <= 65535, "constrain_logits: rows %d unsupported (1..65535)", rows);
    ARG_CHECK(vocab > 0, "constrain_logits: vocab must be positive");
    ARG_CHECK(dtype >= 0 && dtype <= 2, "constrain_logits: dtype %d unknown (0 fp16, 1 bf16, 2 fp32)", dtype);
    ARG_CHECK(logits, "constrain_logits: null pointer (logits)");
    ARG_CHECK(bitmask || bias_offsets, "constrain_logits: neither a bitmask nor a bias given");
    ARG_CHECK(!bias_offsets || (bias_ids && bias_values), "constrain_logits: null pointer (bias_ids / bias_values with bias_offsets)");
    const int words = (int)(((long long)vocab + 31) / 32);
    ARG_CHECK(!bitmask || mask_stride >= words, "constrain_logits: mask_stride %d < ceil(vocab / 32) = %d", mask_stride, words);
    ConstrainParams p{};
    p.logits = logits;
    p.bitmask = reinterpret_cast<const uint32_t*>(bitmask);
    p.bias_offsets = bias_offsets;
    p.bias_ids = bias_ids;
    p.bias_values = bias_values;
    p.vocab = vocab;
    p.mask_stride = mask_stride;
    const dim3 grid((words + kConstrainThreads - 1) / kConstrainThreads, rows);
    auto launch = [&](auto t) {
        return launch_or_record("constrain_logits_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(constrain_logits_kernel<decltype(t)>, {grid, dim3(kConstrainThreads), 0, s, pdl}, p);
        });
    };
    return dtype == 2 ? launch(0.f) : by_dtype(dtype == 1, launch);
}

// ------------------------------------------------------------------------------------------------ peer all-reduce
size_t b200_peer_ar_region_bytes(size_t max_message_bytes) {
    return 2 * peer_strides(max_message_bytes).parity + kArMaxCtas * sizeof(uint32_t) + 256;
}

int b200_peer_alloc(size_t bytes, void** ptr, void* ipc_handle_out /*64 bytes*/) {
    ARG_CHECK(ptr && ipc_handle_out && bytes > 0, "peer_alloc: bad argument");
    void* d = nullptr;
    CUDA_CHECK(cudaMalloc(&d, bytes));
    CUDA_CHECK(cudaMemset(d, 0, bytes));
    CUDA_CHECK(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    CUDA_CHECK(cudaIpcGetMemHandle(&h, d));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(ipc_handle_out, &h, sizeof(h));
    *ptr = d;
    return B200_OK;
}

int b200_peer_open(const void* ipc_handle /*64 bytes*/, void** ptr) {
    ARG_CHECK(ipc_handle && ptr, "peer_open: null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle, sizeof(h));
    void* d = nullptr;
    CUDA_CHECK(cudaIpcOpenMemHandle(&d, h, cudaIpcMemLazyEnablePeerAccess));
    *ptr = d;
    return B200_OK;
}

int b200_peer_allreduce(const void* in, void* out, size_t bytes, int is_bf16, void* const* regions, size_t max_message_bytes,
                        int call_parity, int rank, int world, void* stream) {
    (void)call_parity;   // since r02 the slot parity comes from the device-side call counter (graph replays of any length are safe)
    ARG_CHECK(in && out && regions, "peer_allreduce: null pointer");
    ARG_CHECK(valid_peer_group(rank, world), "peer_allreduce: bad rank/world %d/%d", rank, world);
    ARG_CHECK(bytes > 0 && bytes % 16 == 0 && bytes <= max_message_bytes, "peer_allreduce: message of %zu bytes unsupported", bytes);
    ARG_CHECK((((uintptr_t)in | (uintptr_t)out) & 15) == 0, "peer_allreduce: in/out must be 16-byte aligned");
    PeerArParams p{};
    p.in = in;
    p.out = out;
    int rc = fill_ar_params(p, regions, max_message_bytes, rank, world);
    if (rc) return rc;
    p.n16 = (int)(bytes / 16);
    // W >= 3: reduce-scatter + all-gather (2 hops, (W-1)/W of the volume twice); W == 2: one hop. Env override for tests.
    const int two_shot = env_int("B200_AR_TWOSHOT", world >= 3 ? 1 : 0) && (p.n16 % world == 0);
    // one shot: ~2 chunks (32 B of payload) per thread; two shots: one chunk of the rank's 1/W share per thread
    int ctas = two_shot ? (p.n16 / world + kArThreads - 1) / kArThreads : (p.n16 + 2 * kArThreads - 1) / (2 * kArThreads);
    if (ctas < 1) ctas = 1;
    if (ctas > kArMaxCtas) ctas = kArMaxCtas;
    return by_dtype(is_bf16, [&](auto t) {
        using T = decltype(t);
        return launch_or_record(two_shot ? "peer_allreduce_twoshot_kernel" : "peer_allreduce_kernel", stream,
                                [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(two_shot ? peer_allreduce_twoshot_kernel<T> : peer_allreduce_kernel<T>,
                             {dim3(ctas), dim3(kArThreads), 0, s, pdl}, p);
        });
    });
}

static int allreduce_norm_impl(const void* in, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                               float eps, void* const* regions, size_t max_message_bytes, int rank, int world, int pushed,
                               void* stream) {
    ARG_CHECK(in && residual && gamma && y && regions, "peer_allreduce_norm: null pointer");
    ARG_CHECK(valid_peer_group(rank, world), "peer_allreduce_norm: bad rank/world %d/%d", rank, world);
    ARG_CHECK(rows > 0 && rows <= 65535, "peer_allreduce_norm: rows %d unsupported", rows);
    ARG_CHECK(hidden > 0 && hidden % (8 * world) == 0 && hidden <= 8192, "peer_allreduce_norm: hidden %d must be a multiple of 8*world and <= 8192", hidden);
    ARG_CHECK((size_t)rows * hidden * 2 <= max_message_bytes, "peer_allreduce_norm: message of %zu bytes exceeds the region", (size_t)rows * hidden * 2);
    ARG_CHECK((((uintptr_t)in | (uintptr_t)residual | (uintptr_t)gamma | (uintptr_t)y) & 15) == 0, "peer_allreduce_norm: pointers must be 16-byte aligned");
    PeerArParams p{};
    p.in = in;
    int rc = fill_ar_params(p, regions, max_message_bytes, rank, world);
    if (rc) return rc;
    p.residual = residual;
    p.gamma = gamma;
    p.y = y;
    p.rows = rows;
    p.hidden = hidden;
    p.eps = eps;
    p.pushed = pushed;
    const size_t smem = (size_t)hidden * sizeof(float) + (size_t)(hidden / 8 / world) * 16;
    return by_dtype(is_bf16, [&](auto t) {
        return launch_or_record("peer_allreduce_norm_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(peer_allreduce_norm_kernel<decltype(t)>, {dim3(rows), dim3(kArThreads), smem, s, pdl}, p);
        });
    });
}

int b200_peer_allreduce_norm(const void* in, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                             float eps, void* const* regions, size_t max_message_bytes, int rank, int world, void* stream) {
    return allreduce_norm_impl(in, residual, gamma, y, is_bf16, rows, hidden, eps, regions, max_message_bytes, rank, world, 0, stream);
}
int b200_peer_gather_norm(const void* in, void* residual, const void* gamma, void* y, int is_bf16, int rows, int hidden,
                          float eps, void* const* regions, size_t max_message_bytes, int rank, int world, void* stream) {
    return allreduce_norm_impl(in, residual, gamma, y, is_bf16, rows, hidden, eps, regions, max_message_bytes, rank, world, 1, stream);
}

int b200_peer_argmax(const void* logits, int is_bf16, int rows, int vocab_local, int vocab_total, int32_t* out,
                     void* const* regions, size_t max_message_bytes, int rank, int world, void* stream) {
    ARG_CHECK(logits && out && regions, "peer_argmax: null pointer");
    ARG_CHECK(valid_peer_group(rank, world), "peer_argmax: bad rank/world %d/%d", rank, world);
    ARG_CHECK(rows > 0 && (size_t)rows * 16 <= max_message_bytes && vocab_local > 0 && vocab_total > 0, "peer_argmax: bad shape");
    PeerArParams p{};
    int rc = fill_ar_params(p, regions, max_message_bytes, rank, world);
    if (rc) return rc;
    p.logits = logits;
    p.token_out = out;
    p.rows = rows;
    p.vocab_local = vocab_local;
    p.vocab_total = vocab_total;
    return by_dtype(is_bf16, [&](auto t) {
        return launch_or_record("peer_argmax_kernel", stream, [=, pdl = g_pdl.load() != 0](cudaStream_t s) {
            return launch_ex(peer_argmax_kernel<decltype(t)>, {dim3(rows), dim3(kArThreads), 0, s, pdl}, p);
        });
    });
}

// ------------------------------------------------------------------------------------------------ decode programs
int b200_program_create(b200_program** out) {
    ARG_CHECK(out, "program_create: null pointer");
    *out = new b200_program();
    return B200_OK;
}

int b200_program_begin(b200_program* p) {
    ARG_CHECK(p && !p->finalized, "program_begin: null or already finalised program");
    ARG_CHECK(!g_rec, "program_begin: this thread is already recording a program");
    g_rec = p;
    return B200_OK;
}

int b200_program_end(b200_program* p) {
    ARG_CHECK(p && g_rec == p, "program_end: this thread is not recording this program");
    g_rec = nullptr;
    if (!p->ops.empty()) {
        CUDA_CHECK(cudaMalloc(&p->d_ops, p->ops.size() * sizeof(ProgOp)));
        CUDA_CHECK(cudaMemcpy(p->d_ops, p->ops.data(), p->ops.size() * sizeof(ProgOp), cudaMemcpyHostToDevice));
    }
    const size_t bar_bytes = (p->items.size() + 1) * 256;
    CUDA_CHECK(cudaMalloc(&p->d_bar, bar_bytes));
    CUDA_CHECK(cudaMemset(p->d_bar, 0, bar_bytes));
    CUDA_CHECK(cudaDeviceSynchronize());
    p->finalized = true;
    return B200_OK;
}

int b200_program_set_trace(b200_program* p, void* device_buffer) {
    ARG_CHECK(p, "program_set_trace: null program");
    p->trace = reinterpret_cast<unsigned long long*>(device_buffer);
    return B200_OK;
}

int b200_program_num_ops(const b200_program* p) { return p ? (int)p->ops.size() : 0; }
int b200_program_num_launches(const b200_program* p) { return p ? (int)p->items.size() : 0; }

int b200_program_launch(b200_program* p, void* stream) {
    ARG_CHECK(p && p->finalized, "program_launch: program not finalised (b200_program_end)");
    ARG_CHECK(!g_rec, "program_launch: cannot launch while recording");
    const bool pdl = g_pdl.load() != 0;
    for (size_t i = 0; i < p->items.size(); ++i) {
        const b200_program::Item& it = p->items[i];
        int rc;
        if (it.segment) {
            const bool bf16 = it.bf16 > 0;
            const int bpad = it.bpad > 0 ? it.bpad : 32, qfmt = it.qfmt > 0 ? it.qfmt : B200_FMT_INT4;
            int grid = 0;
            rc = by_dtype(bf16, [&](auto t) { return segment_grid<decltype(t)>(bpad, qfmt, &grid); });
            if (rc) return rc;
            unsigned long long* tr = p->trace ? p->trace + (size_t)it.first * grid * 2 : nullptr;
            // fine timeline (CTA 0): after the coarse region, [op][kFtSlots][kFtBlocks]
            g_ftrace_next = p->trace ? p->trace + p->ops.size() * (size_t)grid * 2 + (size_t)it.first * kFtSlots * kFtBlocks : nullptr;
            rc = by_dtype(bf16, [&](auto t) {
                return launch_segment<decltype(t)>(bpad, qfmt, p->d_ops + it.first, it.count, p->d_bar + i * 64, grid, pdl, tr,
                                                   (cudaStream_t)stream);
            });
            g_ftrace_next = nullptr;
        } else {
            rc = launch_or_record(it.name, stream, it.issue);   // not recording (checked above): launches now
        }
        if (rc) return rc;
    }
    return B200_OK;
}

int b200_program_destroy(b200_program* p) {
    if (!p) return B200_OK;
    if (g_rec == p) g_rec = nullptr;
    if (p->d_ops) cudaFree(p->d_ops);
    if (p->d_bar) cudaFree(p->d_bar);
    delete p;
    return B200_OK;
}

}  // extern "C"
