// Paged GQA decode attention for sm_90a.
//
// Replaces (same math, same cache layout, same page-list format):
//   runXqa                      rtp_llm/models_py/bindings/cuda/ops/CudaXqa.h:65-84 (+CudaXqa.cc:124-221)
//   XQA sm_90a kernel           3rdparty/xqa/mha_sm90.cu
//   FlashInferTRTLLMDecodeOp    rtp_llm/models_py/modules/factory/attention/cuda_impl/trtllm_gen.py:503-546
//
// Work decomposition (not a port of XQA's warpgroup pipeline):
//   grid = (nsplit, B*Hkv); one CTA owns (sequence b, kv head, a contiguous run of 64-token tiles).
//   Warp 4 lane 0 = TMA producer: reads the K/V page ids of each tile from the page list and issues 4-D tensor-map
//   loads (128-byte swizzle, one box per page and per 64-channel half) into a 3-stage shared-memory ring.
//   Warps 0-3 = consumers: each takes 16 of the tile's 64 tokens, S = Q.K^T and O += P.V on the legacy tensor path
//   (ldmatrix + mma.sync m16n8k16; the whole GQA group is packed into the MMA M dimension so every K/V byte is read
//   from HBM exactly once), online softmax with quad-level shuffles, private running (m, l, O) per warp, merged
//   through shared memory at the end.  Sequence splits are merged by the last-arriving CTA (semaphore), XQA-style.
//   Query rows (group x q_len, up to 64) span RT = 1 / 2 / 4 row tiles of 16: consumer warp w owns row tile w % RT and,
//   within each 64-token stage, the 16-token slices w / RT + k * (4 / RT) one after another, so K/V are still read from
//   HBM once per (sequence, kv head) and a warp's registers are those of one row tile. RT == 1 is the single-tile kernel.
//   The kernel is HBM-bound: per CTA 96 KB of K/V in flight, two CTAs per SM.
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace b200 {

constexpr int kAttnTile = 64;          // tokens per pipeline stage
constexpr int kAttnStages = 3;
constexpr int kAttnD = 128;            // head dim
constexpr int kAttnConsumerWarps = 4;
constexpr int kAttnMaxRows = 64;       // query rows (group x q_len) per (sequence, kv head): four 16-row MMA tiles
constexpr int kAttnThreads = (kAttnConsumerWarps + 1) * 32;
// per head dim D (64 / 128 / 256): a stage holds the D/64 64-channel halves of K, then those of V, 8 KB each (64 tokens x 128 B)
__host__ __device__ constexpr int attn_stage_bytes(int D) { return 2 * (D / 64) * kAttnTile * 128; }
__host__ __device__ constexpr int attn_smem_bytes(int D) {
    return kAttnStages * attn_stage_bytes(D) + 1024 /*align*/ + 256 /*barriers etc*/ + 512 /*rope cos/sin table*/;
}
constexpr int kAttnSmemBytes = attn_smem_bytes(kAttnD);

struct AttnParams {
    const void* q;            // [B][Hq][D]
    void* out;                // [B][Hq*D]
    const int32_t* page_list; // [B][1][2][M]
    const int32_t* seq_lens;  // [B] tokens already cached (the new token sits at this index)
    int B, Hq, Hkv, group, M;
    int q_len;                // query tokens per sequence (1 = plain decode; > 1 = verification of speculative tokens, XQA's
                              // max_q_len / trtllm-gen's q_len_per_req): q [B][q_len][Hq][D], query j attends to positions
                              // 0 .. seq_lens[b] + j, its GQA rows sit at MMA rows j * group + g (group * q_len <= 64,
                              // row tile (j * group + g) / 16)
    int T, log2T;             // tokens per page
    int box_h, boxes_per_tile;
    int nsplit, tiles_per_split;
    float scale_log2;         // q_scale * D^-1/2 * log2(e)
    float* ws_o;              // [B*Hkv][nsplit][group][D]
    float* ws_ml;             // [B*Hkv][nsplit][group][2]
    int* sem;                 // [B*Hkv], zero on entry, zero on exit
    // fused RoPE + KV append (XQA's USE_INPUT_KV + ROPE_STYLE, 3rdparty/xqa/mha.h:82-86): when qkv != null the kernel reads the
    // un-rotated q | k | v of the new token from the qkv GEMM output [B][(Hq+2Hkv)*D], rotates q on load, and the CTA that owns
    // the tile of position seq_lens[b] rotates k and appends k, v to the paged cache before streaming it. Same arithmetic as
    // rope_append_kernel (RopeStyle::Base, NeoX pairing) -> bit-identical cache contents and attention output.
    const void* qkv;
    void* kv_pool_rw;
    float log2_base;
    int cluster_merge;        // 1: the nsplit (<= 8) CTAs of a (sequence, kv head) form a thread-block cluster (nsplit,1,1) and merge
                              //    their partial (m, l, O) through distributed shared memory; no workspace, no semaphore
};

// The beam instance's parameters (XQA's beamWidth, 3rdparty/xqa/mha_sm90.cu: ctaNbValidQHeads = headGrpSize * beamWidth). A CTA
// owns a chunk: up to beam_width members, rows of q / out / page_list / seq_lens whose group * beam_width <= 64 query rows share
// it; MMA row i * group + g is member i, head kvh * group + g. q_len is 1.
// Beam mode (chunk_rows null): chunk b is request b, its members the beam_width rows b * beam_width + i; B counts requests.
// Prefix mode: chunk c's members are the rows chunk_rows[chunk_offsets[c] .. chunk_offsets[c + 1]) of the B rows, at most
// beam_width of them (more are cut off); a member row outside [0, B) is skipped (never read or written), and so is a row in no chunk.
struct AttnBeamParams : AttnParams {
    int beam_width;
    const int32_t* shared_lens;   // [chunks] tokens that all members of chunk c share: over the first shared_lens[c] / T pages the
                                  // members' page_list rows are equal (the caller's contract). The kernel rounds it down to whole
                                  // 64-token tiles below the shortest member's cached length, so a wrong value can only cost sharing.
    const int32_t* chunk_offsets; // [chunks + 1]
    const int32_t* chunk_rows;    // [B] (B <= 65535), or null (beam mode)
};

// The tree instance's parameters (a speculative token tree, XQA's spec-decoding mask in TensorRT-LLM). The q_len new tokens of
// sequence b are the nodes of a tree: parents [B][q_len], node 0 the root, node j >= 1 under parents[b][j] in [0, j). Query j
// attends to positions 0 .. seq_lens[b] - 1 and to the slots seq_lens[b] + i of the nodes i on its ancestor walk (itself, its
// parent, ... until the root or a parent outside [0, i)). A chain (parents[j] = j - 1) is the causal q_len instance.
struct AttnTreeParams : AttnParams {
    const int32_t* tree_parents;
};

// RT: 16-row tiles of query rows (rows = group * q_len rounded up to 16 / 32 / 64)
// BEAM: a chunk's members (a request's beams, or rows that share a prefix) in one CTA. Tile t below the shared length is one
// pipeline stage, loaded once through member 0's pages with every row live; a tile from there on is one stage per member that
// reaches it, in member order, each loaded through that member's pages and masked to that member's rows. A row so meets the tiles
// of its own sequence in order with the arithmetic of the plain instance; another member's stage leaves its (m, l, O) bit for bit
// as they were.
// TREE: the q_len instance with each query's new-token columns masked to its ancestors. The ancestor sets are 64-bit masks built
// once per CTA in shared memory. A 16-token slice wholly below seq_lens[b] runs the plain instance's code; a slice that reaches
// the new tokens also tests the mask and reads the new tokens' non-finite V elements as 0, so a node outside a row's ancestors
// never changes that row's bits (p = 0 does not stop 0 * NaN in the mma). A row whose ancestors hold such an element ends NaN.
template <typename T, int D = kAttnD, int RT = 1, bool BEAM = false, bool TREE = false>
__global__ void __launch_bounds__(kAttnThreads, D <= 128 ? 2 : 1)
paged_decode_attn_kernel(const __grid_constant__ CUtensorMap kv_map,
                         const std::conditional_t<BEAM, AttnBeamParams, std::conditional_t<TREE, AttnTreeParams, AttnParams>> p) {
    constexpr int NH = D / 64;                       // 64-channel halves per K / V row
    constexpr int STAGE = attn_stage_bytes(D);
    constexpr int OROW = D + 8;                      // floats; +8 banks per row -> conflict-free float2 stores
    constexpr int NW = kAttnConsumerWarps / RT;      // warps per row tile (each takes RT of a stage's 4 slices)
    static_assert(D == 64 || D == 128 || D == 256, "head_dim 64 / 128 / 256");
    static_assert(RT == 1 || RT == 2 || RT == 4, "1, 2 or 4 row tiles");
    static_assert(!(BEAM && TREE), "a beam step has one query token");
    // the merge staging (per-warp o / m / l, then the cluster partial [rows][D] + (m, l)) reuses the K/V ring
    static_assert((kAttnConsumerWarps * 16 * (OROW + 2) + RT * 16 * (D + 2)) * 4 <= kAttnStages * STAGE,
                  "merge staging exceeds the K/V ring");
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B-swizzled boxes
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kAttnStages * STAGE);
    uint64_t* empty_bar = full_bar + kAttnStages;
    int* s_flag = reinterpret_cast<int*>(empty_bar + kAttnStages);
    float2* cs_tab = reinterpret_cast<float2*>(smem + kAttnStages * STAGE + 256);   // fused rope: (cos, sin) of the 64 channel pairs

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int split = blockIdx.x, bh = blockIdx.y;
    const int b = bh / p.Hkv, kvh = bh % p.Hkv;
    pdl_launch_dependents();   // let the o-projection GEMM start prefetching its weights
    pdl_wait();                // q and the appended K/V come from the previous kernel

    // the host sized the split for max_seq_len: a longer sequence is clamped to that bound (never more tiles than the
    // splits cover, so the last-arriver count below always matches the CTAs that really contribute)
    // query slots per CTA: tokens of a verification step, or the chunk's member slots (BEAM)
    auto nq = [&] {
        if constexpr (BEAM) return p.beam_width;
        else return p.q_len;
    };
    int len_v, sh_tiles = 0;     // BEAM: len is the longest member's, tiles [0, sh_tiles) are shared
    // BEAM: every member's clamped length, then the shared tile count, then (prefix mode) every member's row (kNoRow: a slot
    // past the chunk's members or a row outside [0, B)), in the fused rope's table (the beam instance has no rope)
    int* s_len = reinterpret_cast<int*>(cs_tab);
    uint16_t* s_row = reinterpret_cast<uint16_t*>(s_len + kAttnMaxRows + 1);
    constexpr uint16_t kNoRow = 0xffff;   // (the host keeps B <= 65535 in prefix mode)
    if constexpr (BEAM) {
        const int cap = p.nsplit * p.tiles_per_split * kAttnTile;
        int lmax = 0, cmin = cap;
        // prefix mode: the chunk's rows are chunk_rows[lo, hi), at most beam_width of them; every position read lies in [0, B)
        int lo = 0, nmem = nq();
        if (p.chunk_rows) {
            lo = min(max(p.chunk_offsets[b], 0), p.B);
            nmem = min(min(max(p.chunk_offsets[b + 1], lo), p.B) - lo, p.beam_width);
            if (threadIdx.x == 0) s_flag[1] = lo;   // the workspace merge's position of member 0
        }
        for (int i = lane; i < nq(); i += 32) {
            int row = b * nq() + i;
            if (p.chunk_rows) {
                row = i < nmem ? p.chunk_rows[lo + i] : -1;
                if (row >= p.B) row = -1;
                if (warp == 0) s_row[i] = row < 0 ? kNoRow : (uint16_t)row;
                if (i >= nmem) {                    // an empty slot takes no part
                    if (warp == 0) s_len[i] = 0;
                    continue;
                }
            }
            const int cached = row < 0 ? 0 : min(p.seq_lens[row], cap);
            const int l = row < 0 ? 0 : min(cached + 1, cap);   // a skipped member has no tile of its own and shares nothing
            if (warp == 0) s_len[i] = l;     // (read after the barrier below)
            lmax = max(lmax, l);
            cmin = min(cmin, cached);   // the token appended this step is never shared
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
            cmin = min(cmin, __shfl_xor_sync(0xffffffffu, cmin, o));
        }
        len_v = lmax;
        sh_tiles = min(max(p.shared_lens[b], 0), cmin) / kAttnTile;
        if (threadIdx.x == 0) s_len[kAttnMaxRows] = sh_tiles;   // the stage loops read it from there: a register less to hold
    } else {
        len_v = min(p.seq_lens[b] + p.q_len, p.nsplit * p.tiles_per_split * kAttnTile);
    }
    const int len = len_v;
    const int rows = p.group * nq();
    const int ntiles = (len + kAttnTile - 1) / kAttnTile;
    const int t0 = split * p.tiles_per_split;
    const int t1 = min(t0 + p.tiles_per_split, ntiles);
    const bool empty = t0 >= t1;                 // this split holds no tokens of this sequence (uniform for the CTA)
    if (empty && !p.cluster_merge) return;
    const int nact = (ntiles + p.tiles_per_split - 1) / p.tiles_per_split;  // CTAs that contribute to (b, kvh)

    if (threadIdx.x == 0) {
        for (int s = 0; s < kAttnStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kAttnConsumerWarps);
        }
        fence_mbar_init();
    }
    // TREE: node j's ancestor set (bit i = node i, j's own bit included), in the fused rope's table (the tree instance has no rope)
    uint64_t* s_anc = reinterpret_cast<uint64_t*>(cs_tab);
    if constexpr (TREE) {
        const int j = threadIdx.x;
        if (j < p.q_len) {
            const int32_t* par = p.tree_parents + (size_t)b * p.q_len;
            uint64_t m = 1ull << j;
            for (int i = j; i > 0;) {        // a parent outside [0, i) ends the walk: at most j steps, every read inside the row
                const int pi = par[i];
                if (pi < 0 || pi >= i) break;
                m |= 1ull << pi;
                i = pi;
            }
            s_anc[j] = m;
        }
    }
    __syncthreads();

    // BEAM: the stage sequence, derived alike by the producer and the consumers. live_from: the first member >= from with a stage
    // at tile t (nq() when none); a shared tile has the one stage, filed under member 0, whose pages it is loaded through.
    auto live_from = [&](int t, int from) {
        if (t < s_len[kAttnMaxRows]) return from == 0 ? 0 : nq();
        while (from < nq() && s_len[from] <= t * kAttnTile) ++from;
        return from;
    };

    if (warp == kAttnConsumerWarps) {
        // ------------------------------------------------------------------ TMA producer
        // Tile issue is split in two so that, with the fused rope, the append of the new token (all 32 lanes) overlaps the first
        // loads in flight: lane 0 first fills the ring with tiles that cannot contain the new token, the warp appends, then
        // lane 0 streams the rest (the token's tile is the sequence's last tile).
        int seq = b;                                  // page_list row
        if constexpr (BEAM) seq = b * nq();             // beam 0's; beam i's rows lie 2 * M * i further on
        const int32_t* kpl = p.page_list + (size_t)(seq * 2 + 0) * p.M;
        const int32_t* vpl = p.page_list + (size_t)(seq * 2 + 1) * p.M;
        // BEAM: stage n of this CTA is tile i through member `beam`'s pages (a live member's row is valid), up to that member's
        // length when the tile is private
        auto issue = [&](int i, int n = 0, int beam = 0) {
            int it = i - t0, len_s = len;
            const int32_t *kp = kpl, *vp = vpl;
            if constexpr (BEAM) {
                it = n;
                if (p.chunk_rows) {
                    kp = p.page_list + (size_t)s_row[beam] * 2 * p.M;
                    vp = kp + p.M;
                } else {
                    kp += (size_t)beam * 2 * p.M;
                    vp += (size_t)beam * 2 * p.M;
                }
                if (i >= s_len[kAttnMaxRows]) len_s = s_len[beam];
            }
            const int s = it % kAttnStages;
            const uint32_t ph = (it / kAttnStages) & 1;
            // page ids first (global loads overlap the wait below)
            int kpage[4], vpage[4], inpage[4];
            int nbox = 0;
#pragma unroll
            for (int bx = 0; bx < 4; ++bx) {
                const int tok = i * kAttnTile + bx * p.box_h;
                if (bx < p.boxes_per_tile && tok < len_s) {
                    const int pidx = tok >> p.log2T;
                    kpage[bx] = kp[pidx];
                    vpage[bx] = vp[pidx];
                    inpage[bx] = tok & (p.T - 1);
                    nbox = bx + 1;
                }
            }
            mbar_wait(&empty_bar[s], ph ^ 1);
            uint8_t* stage = smem + s * STAGE;
            mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(nbox * 2 * NH * p.box_h * 128));
#pragma unroll
            for (int bx = 0; bx < 4; ++bx) {
                if (bx < nbox) {
                    const int row_off = bx * p.box_h * 128;
#pragma unroll
                    for (int h = 0; h < NH; ++h) {
                        tma_load_4d(stage + h * 8192 + row_off, &kv_map, 64 * h, inpage[bx], kvh, kpage[bx], &full_bar[s]);
                        tma_load_4d(stage + (NH + h) * 8192 + row_off, &kv_map, 64 * h, inpage[bx], kvh, vpage[bx], &full_bar[s]);
                    }
                }
            }
        };
        int first_end = t1;                               // tiles [t0, first_end) are issued before the append
        bool own = false;
        int pos = 0;
        if (!BEAM && !TREE && D == 128 && RT == 1 && p.qkv != nullptr) {   // fused rope: head_dim 128, one row tile (the host rejects others)
            pos = p.seq_lens[b];
            own = pos < len && (pos / kAttnTile) >= t0 && (pos / kAttnTile) < t1;      // this CTA streams the new token's tile
            if (own) first_end = min(min(t0 + kAttnStages, t1), pos / kAttnTile);
        }
        if (lane == 0) {
            tma_prefetch_desc(&kv_map);
            if constexpr (BEAM) {
                int n = 0;
                for (int i = t0; i < t1; ++i)
                    for (int beam = live_from(i, 0); beam < nq(); beam = live_from(i, beam + 1)) issue(i, n++, beam);
            } else {
                for (int i = t0; i < first_end; ++i) issue(i);
            }
        }
        __syncwarp();
        if (own) {
            const T* row = reinterpret_cast<const T*>(p.qkv) + (size_t)b * (p.Hq + 2 * p.Hkv) * kAttnD;
            const T* ksrc = row + (size_t)(p.Hq + kvh) * kAttnD;
            const T* vsrc = row + (size_t)(p.Hq + p.Hkv + kvh) * kAttnD;
            const size_t page_elems = (size_t)p.Hkv * p.T * kAttnD;
            const int32_t kpage = kpl[pos >> p.log2T], vpage = vpl[pos >> p.log2T];
            T* pool = reinterpret_cast<T*>(p.kv_pool_rw);
            T* kdst = pool + (size_t)kpage * page_elems + ((size_t)kvh * p.T + (pos & (p.T - 1))) * kAttnD;
            T* vdst = pool + (size_t)vpage * page_elems + ((size_t)kvh * p.T + (pos & (p.T - 1))) * kAttnD;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int i = lane + 32 * j;                        // channel pair (i, i + 64)
                const float x0 = to_f32<T>(ksrc[i]), x1 = to_f32<T>(ksrc[i + 64]);
                const float2 cf = rope_base_cos_sin(i, kAttnD, p.log2_base, pos);
                float r0, r1;
                rope_rotate(x0, x1, cf.x, cf.y, r0, r1);
                kdst[i] = from_f32<T>(r0);
                kdst[i + 64] = from_f32<T>(r1);
                vdst[i] = vsrc[i];
                vdst[i + 64] = vsrc[i + 64];
            }
            __threadfence();              // every lane's stores are performed before lane 0 (after the warp barrier) ...
            fence_proxy_async_global();   // ... issues the TMA loads of the token's tile, which read them through the async proxy
        }
        __syncwarp();
        if (own && lane == 0) fence_proxy_async_global();
        if (lane == 0) {
            for (int i = first_end; i < t1; ++i) issue(i);
        }
        if (!p.cluster_merge) return;  // the producer warp takes no part in the merge (named barrier 1 counts 128 threads)
        cluster_sync_all();            // ... but every thread of the cluster passes the two cluster barriers of the DSMEM merge
        cluster_sync_all();
        return;
    }

    // ---------------------------------------------------------------------- consumers
    const int qrow = lane >> 2;          // fragment row (and row + 8)
    const int qcol = (lane & 3) * 2;     // fragment column pair
    const int rt = warp % RT;            // this warp's row tile: MMA rows rt * 16 + qrow (and + 8)
    const int row0 = rt * 16 + qrow, row1 = row0 + 8;
    // Q fragments for the whole head dim: 8 k-steps x 4 regs. Rows >= group are zero.
    uint32_t qf[D / 16][4];
    bool q_loaded = false;
    if constexpr (D == 128 && RT == 1 && !BEAM && !TREE) {
      if (p.qkv) {
        q_loaded = true;
        // un-rotated q straight from the qkv GEMM output; the NeoX partner of column c < 64 is column c + 64 = the same
        // register index four k-steps later, so the rotation stays inside a thread
        const T* qbase = reinterpret_cast<const T*>(p.qkv) + ((size_t)b * (p.Hq + 2 * p.Hkv) + (size_t)kvh * p.group) * kAttnD;
        const bool v0 = qrow < p.group, v1 = (qrow + 8) < p.group;
        const int pos = p.seq_lens[b];
        if (threadIdx.x < 64)                                // one sincosf per channel pair and CTA, shared through smem
            cs_tab[threadIdx.x] = rope_base_cos_sin(threadIdx.x, kAttnD, p.log2_base, pos);
        asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int hc = 0; hc < 2; ++hc) {                 // column groups c and c + 8 of the k-step
                const int c = kk * 16 + qcol + hc * 8;
                const float2 t0c = cs_tab[c], t1c = cs_tab[c + 1];
                const float cs[2] = {t0c.x, t1c.x}, sn[2] = {t0c.y, t1c.y};
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {             // fragment rows qrow and qrow + 8
                    const bool ok = rr ? v1 : v0;
                    uint32_t lo = 0u, hi = 0u;
                    if (ok) {
                        const T* src = qbase + (size_t)(qrow + 8 * rr) * kAttnD + c;
                        const float a0 = to_f32<T>(src[0]), a1 = to_f32<T>(src[1]);          // x0 (columns c, c+1)
                        const float b0 = to_f32<T>(src[64]), b1 = to_f32<T>(src[65]);        // x1 (columns c+64, c+65)
                        float l0r, h0r, l1r, h1r;
                        rope_rotate(a0, b0, cs[0], sn[0], l0r, h0r);
                        rope_rotate(a1, b1, cs[1], sn[1], l1r, h1r);
                        lo = pack2<T>(l0r, l1r);
                        hi = pack2<T>(h0r, h1r);
                    }
                    qf[kk][hc * 2 + rr] = lo;
                    qf[kk + 4][hc * 2 + rr] = hi;
                }
            }
        }
      }
    }
    if (!q_loaded) {
        // MMA row R = j * group + g  <->  query token (BEAM: member) j, head kvh * group + g
        bool v0 = row0 < rows, v1 = row1 < rows;
        if constexpr (BEAM) if (p.chunk_rows) {
            v0 = v0 && s_row[row0 / p.group] != kNoRow;
            v1 = v1 && s_row[row1 / p.group] != kNoRow;
        }
        const T* qall = reinterpret_cast<const T*>(p.q);
        const T* q0 = qall + (((size_t)b * nq() + row0 / p.group) * p.Hq + (size_t)kvh * p.group + row0 % p.group) * D;
        const T* q1 = qall + (((size_t)b * nq() + row1 / p.group) * p.Hq + (size_t)kvh * p.group + row1 % p.group) * D;
        if constexpr (BEAM) if (p.chunk_rows) {   // prefix mode: member j is row s_row[j]
            q0 = qall + ((size_t)s_row[row0 / p.group] * p.Hq + (size_t)kvh * p.group + row0 % p.group) * D;
            q1 = qall + ((size_t)s_row[row1 / p.group] * p.Hq + (size_t)kvh * p.group + row1 % p.group) * D;
        }
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
            const int c = kk * 16 + qcol;
            qf[kk][0] = v0 ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
            qf[kk][1] = v1 ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
            qf[kk][2] = v0 ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
            qf[kk][3] = v1 ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
        }
    }

    float o[D / 8][4];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY;  // running max (raw score units) for rows qrow / qrow+8
    float l0 = 0.f, l1 = 0.f;              // per-thread partial row sums (quad-reduced at the end)
    const float sl2 = p.scale_log2;
    int off0 = 0, off1 = 0;   // (BEAM: one query token per beam; TREE: the ancestor masks stand for the causal offsets)
    int tree_base = 0;        // TREE: seq_lens[b], the position of node 0
    bool pois0 = false, pois1 = false;   // TREE: the row attends to a new token's non-finite V element
    if constexpr (TREE) tree_base = p.seq_lens[b];
    if constexpr (!BEAM && !TREE) {
        off0 = p.q_len - 1 - min(row0 / p.group, p.q_len - 1);
        off1 = p.q_len - 1 - min(row1 / p.group, p.q_len - 1);
    }

    // ldmatrix lane geometry
    const int mi = lane >> 3, mr = lane & 7;
    const int k_tokrow0 = warp / RT * 16 + (mi >> 1) * 8 + mr;  // K: matrices (tok0-7,c),(tok0-7,c+1),(tok8-15,c),(tok8-15,c+1)
    const int k_chunk_add = mi & 1;
    const int v_tokrow0 = warp / RT * 16 + (mi & 1) * 8 + mr;   // V (trans): (tok0-7,c),(tok8-15,c),(tok0-7,c+1),(tok8-15,c+1)
    const int v_chunk_add = mi >> 1;

    // BEAM: the stage's beam and count; in a private stage only the beam's own rows are kept (row0 / row1 of this thread)
    int nstage = 0;
    for (int i = t0; i < t1; ++i) {
      int beam = 0;
      if constexpr (BEAM) beam = live_from(i, 0);
      do {      // (one pass unless BEAM)
        int it = i - t0, len_s = len;
        bool keep0 = true, keep1 = true;
        if constexpr (BEAM) {
            it = nstage++;
            len_s = (i + 1) * kAttnTile;   // a shared tile is whole in every beam
        }
        const int s = it % kAttnStages;
        const uint32_t ph = (it / kAttnStages) & 1;
        mbar_wait(&full_bar[s], ph);
        uint8_t* stage = smem + s * STAGE;
        const uint32_t k_base = smem_u32(stage), v_base = k_base + NH * 8192;
        if constexpr (BEAM) {
            if (i >= s_len[kAttnMaxRows]) {
                len_s = s_len[beam];
                const int r0 = rt * 16 + qrow - beam * p.group;   // row0, counted from the beam's first row
                keep0 = r0 >= 0 && r0 < p.group;
                keep1 = r0 + 8 >= 0 && r0 + 8 < p.group;
                // no row of this beam in the warp's row tile: nothing to compute, but the stage is still this warp's to release
                if (beam * p.group >= rt * 16 + 16 || (beam + 1) * p.group <= rt * 16) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[s]);
                    continue;
                }
            }
        }

      int nks = RT;
      // The beam instances of two and four row tiles keep their slice passes a loop (the count is hidden from the compiler):
      // unrolled, the accumulators a private stage sets aside push them over the register budget of two CTAs per SM (spills).
      if constexpr (BEAM && RT > 1) asm volatile("" : "+r"(nks));
#pragma unroll
      for (int ks = 0; ks < nks; ++ks) {
        const int slice = warp / RT + ks * NW;           // 16-token slice of the stage
        const int k_tokrow = k_tokrow0 + ks * NW * 16, v_tokrow = v_tokrow0 + ks * NW * 16;
        const int tok0 = i * kAttnTile + slice * 16;
        const int valid = len_s - tok0;  // tokens of this slice that exist (may be <= 0)
        if (valid < 16) {
            // Rows past the end of the sequence hold stale / never-written bytes: P is 0 there but 0 * NaN = NaN,
            // so the V rows are zeroed before use (K garbage is masked on the scores below). With RT > 1 the warps of the
            // other row tiles zero the same rows: they all store zeros, and each reads only after its own stores.
            const int first = valid < 0 ? 0 : valid;
            for (int r = first; r < 16; ++r) {
                uint8_t* row = stage + NH * 8192 + (slice * 16 + r) * 128;
#pragma unroll
                for (int h = 0; h < NH; ++h) reinterpret_cast<uint32_t*>(row + h * 8192)[lane] = 0u;
            }
            __syncwarp();
        }

        // ---- S = Q K^T for 16 heads x 16 tokens
        float sc[2][4];
#pragma unroll
        for (int j = 0; j < 2; ++j) sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
            const int half = kk >> 2, c = (kk & 3) * 2 + k_chunk_add;
            uint32_t kb[4];
            ldmatrix_x4(kb, k_base + half * 8192 + k_tokrow * 128 + ((c ^ (k_tokrow & 7)) << 4));
            mma_m16n8k16<T>(sc[0], qf[kk], kb[0], kb[1]);
            mma_m16n8k16<T>(sc[1], qf[kk], kb[2], kb[3]);
        }

        // ---- mask + online softmax (rows qrow and qrow+8)
        float mx0 = -INFINITY, mx1 = -INFINITY;
        int lim0 = valid - off0, lim1 = valid - off1;
        if constexpr (BEAM) {   // another beam's stage: every score of the row is masked
            if (!keep0) lim0 = 0;
            if (!keep1) lim1 = 0;
        }
        // TREE: bit c of vis = column c of the slice is visible to the row (column c is new token rel + c, cached when < 0)
        const int rel = tok0 - tree_base;
        const bool tail = TREE && rel > -16 && rel < kAttnMaxRows;   // the slice reaches the new tokens
        uint32_t vis0 = 0xffffu, vis1 = 0xffffu;
        if constexpr (TREE) if (tail) {
            const uint64_t a0 = s_anc[min(row0 / p.group, p.q_len - 1)], a1 = s_anc[min(row1 / p.group, p.q_len - 1)];
            const uint64_t below = rel < 0 ? (1ull << -rel) - 1 : 0ull;
            vis0 = (uint32_t)((rel >= 0 ? a0 >> rel : (a0 << -rel) | below) & 0xffffu);
            vis1 = (uint32_t)((rel >= 0 ? a1 >> rel : (a1 << -rel) | below) & 0xffffu);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                // query j of a q_len-token step sees q_len - 1 - j fewer tokens than the last one (causal among the new tokens)
                bool ok0 = (j * 8 + qcol + e) < lim0, ok1 = (j * 8 + qcol + e) < lim1;
                if constexpr (TREE) {
                    ok0 = ok0 && ((vis0 >> (j * 8 + qcol + e)) & 1u);
                    ok1 = ok1 && ((vis1 >> (j * 8 + qcol + e)) & 1u);
                }
                sc[j][e] = ok0 ? sc[j][e] : -INFINITY;
                sc[j][2 + e] = ok1 ? sc[j][2 + e] : -INFINITY;
                mx0 = fmaxf(mx0, sc[j][e]);
                mx1 = fmaxf(mx1, sc[j][2 + e]);
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
        // a fully masked slice keeps m = -inf; use 0 as the subtrahend so exp2(-inf - 0) = 0 (no NaN)
        const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0 * sl2, ms1 = (mn1 == -INFINITY) ? 0.f : mn1 * sl2;
        float a0 = fast_exp2(m0 * sl2 - ms0), a1 = fast_exp2(m1 * sl2 - ms1);  // m = -inf -> 0
        if constexpr (BEAM) {
            // A masked row has mn = m and p = 0, but m * sl2 - ms may contract to an fma and leave the product's rounding error in
            // the exponent. Another beam's stage must not rescale the row at all: the sharing a caller declares never changes bits.
            if (!keep0) a0 = 1.f;
            if (!keep1) a1 = 1.f;
        }
        m0 = mn0;
        m1 = mn1;
        float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                sc[j][e] = fast_exp2(fmaf(sc[j][e], sl2, -ms0));
                sc[j][2 + e] = fast_exp2(fmaf(sc[j][2 + e], sl2, -ms1));
                ps0 += sc[j][e];
                ps1 += sc[j][2 + e];
            }
        }
        l0 = fmaf(l0, a0, ps0);
        l1 = fmaf(l1, a1, ps1);
        if (a0 != 1.f || a1 != 1.f) {
#pragma unroll
            for (int n = 0; n < D / 8; ++n) {
                o[n][0] *= a0;
                o[n][1] *= a0;
                o[n][2] *= a1;
                o[n][3] *= a1;
            }
        }
        // P (rounded to the cache element type, 3rdparty/xqa/ref.py:80) as the A fragment of the second product
        uint32_t pf[4];
        pf[0] = pack2<T>(sc[0][0], sc[0][1]);
        pf[1] = pack2<T>(sc[0][2], sc[0][3]);
        pf[2] = pack2<T>(sc[1][0], sc[1][1]);
        pf[3] = pack2<T>(sc[1][2], sc[1][3]);

        // ---- O += P V
        if constexpr (TREE) {
          // (two loops, so that a slice below the new tokens runs the plain loop without a branch between its loads and mmas)
          if (tail) {
            // register vb[r] holds slice tokens (r & 1) * 8 + 2 * (lane & 3) (low half) and + 1 (high half); newv[r & 1] selects the
            // halves of new tokens, whose non-finite elements are read as 0 and recorded in `bad` (bit = slice token)
            uint32_t newv[2], bad = 0u;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int t = h * 8 + 2 * (lane & 3);
                newv[h] = (rel + t >= 0 ? 0x0000ffffu : 0u) | (rel + t + 1 >= 0 ? 0xffff0000u : 0u);
            }
            constexpr uint32_t E = std::is_same<T, __half>::value ? 0x7c00u : 0x7f80u;   // exponent all ones: inf / NaN
#pragma unroll
            for (int n2 = 0; n2 < D / 16; ++n2) {
                const int half = n2 >> 2, c = (n2 & 3) * 2 + v_chunk_add;
                uint32_t vb[4];
                ldmatrix_x4_trans(vb, v_base + half * 8192 + v_tokrow * 128 + ((c ^ (v_tokrow & 7)) << 4));
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const uint32_t x = vb[r];
                    const uint32_t nf = (((x & E) == E ? 0x0000ffffu : 0u) | (((x >> 16) & E) == E ? 0xffff0000u : 0u)) & newv[r & 1];
                    const int t = (r & 1) * 8 + 2 * (lane & 3);
                    bad |= ((nf & 0xffffu) ? 1u << t : 0u) | ((nf >> 16) ? 2u << t : 0u);
                    vb[r] = x & ~nf;
                }
                mma_m16n8k16<T>(o[2 * n2], pf, vb[0], vb[1]);
                mma_m16n8k16<T>(o[2 * n2 + 1], pf, vb[2], vb[3]);
            }
            bad = __reduce_or_sync(0xffffffffu, bad);
            pois0 |= (bad & vis0) != 0u;
            pois1 |= (bad & vis1) != 0u;
          } else {
#pragma unroll
            for (int n2 = 0; n2 < D / 16; ++n2) {
                const int half = n2 >> 2, c = (n2 & 3) * 2 + v_chunk_add;
                uint32_t vb[4];
                ldmatrix_x4_trans(vb, v_base + half * 8192 + v_tokrow * 128 + ((c ^ (v_tokrow & 7)) << 4));
                mma_m16n8k16<T>(o[2 * n2], pf, vb[0], vb[1]);
                mma_m16n8k16<T>(o[2 * n2 + 1], pf, vb[2], vb[3]);
            }
          }
        } else {
#pragma unroll
        for (int n2 = 0; n2 < D / 16; ++n2) {
            const int half = n2 >> 2, c = (n2 & 3) * 2 + v_chunk_add;
            uint32_t vb[4];
            ldmatrix_x4_trans(vb, v_base + half * 8192 + v_tokrow * 128 + ((c ^ (v_tokrow & 7)) << 4));
            if constexpr (BEAM) {
                // p = 0 does not shield a row from another beam's V: 0 * inf and 0 * NaN are NaN. A row the stage does not keep
                // takes its accumulators back as they were.
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float(&acc)[4] = o[2 * n2 + h];
                    const float old[4] = {acc[0], acc[1], acc[2], acc[3]};
                    mma_m16n8k16<T>(acc, pf, vb[2 * h], vb[2 * h + 1]);
                    if (!keep0) acc[0] = old[0], acc[1] = old[1];
                    if (!keep1) acc[2] = old[2], acc[3] = old[3];
                }
            } else {
                mma_m16n8k16<T>(o[2 * n2], pf, vb[0], vb[1]);
                mma_m16n8k16<T>(o[2 * n2 + 1], pf, vb[2], vb[3]);
            }
        }
        }
      }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      } while (BEAM && (beam = live_from(i, beam + 1)) < nq());
    }

    // quad-reduce the row sums
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    if constexpr (TREE) {   // (uniform over the quad: vis and bad are the row's and the warp's)
        if (pois0) l0 = __int_as_float(0x7fffffff);
        if (pois1) l1 = __int_as_float(0x7fffffff);
    }

    // ---------------------------------------------------------------------- merge the NW warps of each row tile through smem
    asm volatile("bar.sync 1, 128;" ::: "memory");  // everyone is done reading the K/V ring
    float* o_s = reinterpret_cast<float*>(smem);                              // [4][16][OROW]
    float* m_s = o_s + kAttnConsumerWarps * 16 * OROW;                        // [4][16]
    float* l_s = m_s + kAttnConsumerWarps * 16;                               // [4][16]
    {
        float* ow = o_s + (size_t)warp * 16 * OROW;
#pragma unroll
        for (int n = 0; n < D / 8; ++n) {
            *reinterpret_cast<float2*>(ow + qrow * OROW + n * 8 + qcol) = make_float2(o[n][0], o[n][1]);
            *reinterpret_cast<float2*>(ow + (qrow + 8) * OROW + n * 8 + qcol) = make_float2(o[n][2], o[n][3]);
        }
        if ((lane & 3) == 0) {
            m_s[warp * 16 + qrow] = m0;
            m_s[warp * 16 + qrow + 8] = m1;
            l_s[warp * 16 + qrow] = l0;
            l_s[warp * 16 + qrow + 8] = l1;
        }
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");

    // thread t finishes the output channels t, t + 128, ... < D
    constexpr int DPT = (D + 127) / 128;
    const int d0 = threadIdx.x;
    // workspace row of MMA row r and split sp. BEAM: member i's partials sit at its position (b * beam_width or chunk_offsets[b]) + i,
    // [B][Hkv][nsplit][group]
    // (B rows, so the workspace of a plain launch on the rows holds them, and a position lies in [0, B) whatever the chunks hold)
    auto ws_row = [&](int r, int sp) -> size_t {
        if constexpr (BEAM)
            return (((size_t)((p.chunk_rows ? s_flag[1] : b * nq()) + r / p.group) * p.Hkv + kvh) * p.nsplit + sp) * p.group + r % p.group;
        else return (size_t)0;   // (not called)
    };
    const size_t ws_base = ((size_t)bh * p.nsplit + split) * rows;
    // output row of MMA row r: token (BEAM: member) r / group, head kvh * group + r % group of out [B][q_len][Hq * D]
    auto out_row = [&](int r) {
        if constexpr (BEAM) if (p.chunk_rows)
            return reinterpret_cast<T*>(p.out) + ((size_t)s_row[r / p.group] * p.Hq + (size_t)kvh * p.group + r % p.group) * D;
        return reinterpret_cast<T*>(p.out) + (((size_t)b * nq() + r / p.group) * p.Hq + (size_t)kvh * p.group + r % p.group) * D;
    };
    // per-CTA partial of the cluster merge: [rows][D] fp32 + (m, l) per row, behind the per-warp staging area
    float* part_o = l_s + kAttnConsumerWarps * 16;
    float* part_ml = part_o + RT * 16 * D;
    for (int r = 0; r < rows; ++r) {
        if constexpr (BEAM) if (p.chunk_rows && s_row[r / p.group] == kNoRow) continue;   // a skipped member's rows are not written
        // row r is row rr of row tile r / 16, staged by the warps w = r / 16 + RT * j (j < NW)
        const int wt = RT == 1 ? 0 : r >> 4, rr = RT == 1 ? r : r & 15;
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < NW; ++j) m = fmaxf(m, m_s[(wt + RT * j) * 16 + rr]);
        float f[NW], l = 0.f;
#pragma unroll
        for (int j = 0; j < NW; ++j) {
            f[j] = (m == -INFINITY) ? 0.f : fast_exp2((m_s[(wt + RT * j) * 16 + rr] - m) * sl2);  // -inf -> 0
            l = fmaf(f[j], l_s[(wt + RT * j) * 16 + rr], l);
        }
        if (d0 == 0) {
            if (p.cluster_merge) {
                part_ml[r * 2 + 0] = m;
                part_ml[r * 2 + 1] = l;
            } else if (nact > 1) {
                p.ws_ml[(BEAM ? ws_row(r, split) : ws_base + r) * 2 + 0] = m;
                p.ws_ml[(BEAM ? ws_row(r, split) : ws_base + r) * 2 + 1] = l;
            }
        }
#pragma unroll
        for (int j = 0; j < DPT; ++j) {
            const int d = d0 + 128 * j;
            if (d >= D) break;
            float acc = 0.f;
#pragma unroll
            for (int w = 0; w < NW; ++w) acc = fmaf(f[w], o_s[((size_t)(wt + RT * w) * 16 + rr) * OROW + d], acc);
            if (p.cluster_merge) part_o[r * D + d] = acc;
            else if (nact == 1) out_row(r)[d] = from_f32<T>(acc / l);
            else p.ws_o[(BEAM ? ws_row(r, split) : ws_base + r) * D + d] = acc;
        }
    }
    if (p.cluster_merge) {
        // ---------------------------------------------------------------------- cross-CTA merge through DSMEM
        // CTA `rank` of the cluster (= split) finishes the GQA rows r = rank, rank + nsplit, ...: every row is reduced by
        // exactly one CTA in fixed split order 0..nsplit-1 (deterministic); empty splits carry m = -inf, l = 0.
        cluster_sync_all();
        const int S = p.nsplit;
        const uint32_t o_addr = smem_u32(part_o), ml_addr = smem_u32(part_ml);
        for (int r = (int)cluster_ctarank(); r < rows; r += S) {
            if constexpr (BEAM) if (p.chunk_rows && s_row[r / p.group] == kNoRow) continue;
            float mm[8], ll[8];
            float m = -INFINITY;
#pragma unroll
            for (int sp = 0; sp < 8; ++sp) {
                if (sp < S) {
                    mm[sp] = dsmem_ld_f32(dsmem_addr(ml_addr + (r * 2 + 0) * 4, sp));
                    ll[sp] = dsmem_ld_f32(dsmem_addr(ml_addr + (r * 2 + 1) * 4, sp));
                    m = fmaxf(m, mm[sp]);
                }
            }
            float l = 0.f;
#pragma unroll
            for (int sp = 0; sp < 8; ++sp) {
                if (sp < S) {
                    mm[sp] = fast_exp2((mm[sp] - m) * sl2);      // -inf -> 0 (m is finite: the sequence has >= 1 token)
                    l = fmaf(mm[sp], ll[sp], l);
                }
            }
#pragma unroll
            for (int j = 0; j < DPT; ++j) {
                const int d = d0 + 128 * j;
                if (d >= D) break;
                float oo[8];
#pragma unroll
                for (int sp = 0; sp < 8; ++sp)
                    if (sp < S) oo[sp] = dsmem_ld_f32(dsmem_addr(o_addr + (r * D + d) * 4, sp));
                float acc = 0.f;
#pragma unroll
                for (int sp = 0; sp < 8; ++sp)
                    if (sp < S) acc = fmaf(mm[sp], oo[sp], acc);
                out_row(r)[d] = from_f32<T>(acc / l);
            }
        }
        cluster_sync_all();   // peers may still be reading this CTA's partial
        return;
    }
    if (nact == 1) return;

    // ---------------------------------------------------------------------- cross-CTA merge: last arriver reduces
    __threadfence();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (threadIdx.x == 0) {
        const int prev = atomicAdd(&p.sem[bh], 1);
        *s_flag = (prev == nact - 1);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (!*s_flag) return;
    __threadfence();
    for (int r = 0; r < rows; ++r) {
        if constexpr (BEAM) if (p.chunk_rows && s_row[r / p.group] == kNoRow) continue;
        float m = -INFINITY;
        for (int sp = 0; sp < nact; ++sp)
            m = fmaxf(m, __ldcg(&p.ws_ml[(BEAM ? ws_row(r, sp) : ((size_t)bh * p.nsplit + sp) * rows + r) * 2 + 0]));
#pragma unroll
        for (int j = 0; j < DPT; ++j) {
            const int d = d0 + 128 * j;
            if (d >= D) break;
            float acc = 0.f, l = 0.f;
            for (int sp = 0; sp < nact; ++sp) {
                const size_t row = BEAM ? ws_row(r, sp) : ((size_t)bh * p.nsplit + sp) * rows + r;
                const float fsp = fast_exp2((__ldcg(&p.ws_ml[row * 2 + 0]) - m) * sl2);
                acc = fmaf(fsp, __ldcg(&p.ws_o[row * D + d]), acc);
                l = fmaf(fsp, __ldcg(&p.ws_ml[row * 2 + 1]), l);
            }
            out_row(r)[d] = from_f32<T>(acc / l);
        }
    }
    if (threadIdx.x == 0) p.sem[bh] = 0;  // self-reset for the next launch
}

}  // namespace b200
