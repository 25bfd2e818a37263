// Tensor-core (wgmma) candidate pass of the evaluator for large catalogues
// (BASELINE config 4: 1 M users x 10 M items x d=128, SURVEY.md 7.1 "tensor-core path").
//
// Replaces the score step of evaluator/backend/cpp/uni_evaluator.py:134 (model.predict = U.V^T,
// MF.py:120-122) for catalogues where an fp32 SIMT contraction is far off the machine's
// throughput.  The ranking still has to be the reference's, bit for bit, so the tensor cores
// only SELECT: scores are computed from bf16 copies of the tables (exact products, fp32
// accumulation), every item whose approximate score can still belong to the exact top K+1 (a
// rigorous margin, see tc_prepare_users_kernel) becomes a candidate, and the candidates are
// re-scored with the oracle's fp32 FMA chain and ranked by the tie-aware selection of evaluator.cu
// (users with ties: second pass with the reference's heap root as threshold + libstdc++ heap replay).
//
// Hopper (sm_90a) features used here:
//   * TMA: cp.async.bulk.tensor.2d through a CUtensorMap (SWIZZLE_128B, NT x 64 bf16 boxes, rows
//     past the end of the table zero-filled) brings the item tiles into a ring of shared-memory
//     stages; completion is signalled with mbarrier complete_tx;
//   * wgmma.mma_async m64 x N{64|128} x k16, bf16 in, fp32 accumulators in registers; each of the
//     two consumer warpgroups owns 64 users, both operands come from shared memory through
//     matrix descriptors (K-major, SWIZZLE_128B: 64-element K blocks, rows 128 B apart, 16-byte
//     chunk c of row r at c ^ (r & 7));
//   * the accumulators are staged through shared memory so that the filter keeps one user per
//     thread and visits the items of its list in ascending order.
// The kernel and its pipeline are described above tc_candidate_kernel and in DESIGN.md section 3a;
// nrc_tc_gemm_debug below is the stand-alone MMA building block the tests use to pin the
// descriptor encodings (no-swizzle and SWIZZLE_128B) against a torch matmul.
#include <cuda.h>            // CUtensorMap (types only; the encoder is fetched from the driver at run time)
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace nrc {
namespace tc {

constexpr int kWgM = 64;       // users per warpgroup (wgmma M)
constexpr int kMmaK = 16;      // bf16 elements per wgmma k-step

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// TMA: one [box_rows x 64] bf16 box of a row-major [rows, K] tensor -> shared memory, laid out
// by the copy engine in the SWIZZLE_128B pattern the wgmma descriptors below expect; rows past
// the end of the tensor arrive as zeros.  Completion is signalled on `bar` (complete_tx).
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int c_k, int c_row, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c_k), "r"(c_row), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// shared-memory writes made with ordinary stores must be fenced before the tensor core (async
// proxy) reads them
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma ordering: fence before the first wgmma that touches registers written by ordinary
// instructions; commit the issued wgmmas as one group and wait for it
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// the accumulator registers are in/out operands so that no use of them is scheduled above the wait
template <int R>
__device__ __forceinline__ void wgmma_keep(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// named barrier of one warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// wgmma shared-memory matrix descriptor (sm_90a): [0,14) start>>4, [16,30) LBO>>4, [32,46) SBO>>4,
// [62,64) layout: 0 = no swizzle (8 x 16-byte core matrices), 1 = SWIZZLE_128B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout_type = 0) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)(layout_type & 3u) << 62;
    return d;
}

// SWIZZLE_128B K-major layout: the tile is cut along K into blocks of 64 bf16 (128 B); inside a
// block row r occupies 128 contiguous bytes at r*128 and its 16-byte chunk c sits at position
// c ^ (r & 7); 8-row groups are 1024 B apart (SBO), LBO is unused (1).  A warp copying 4 rows x 8
// chunks reads 4 x 128 contiguous global bytes and stores conflict-free.
__device__ __forceinline__ void load_tile_sw128(uint8_t* smem, const __nv_bfloat16* __restrict__ g, int rows,
                                                int valid_rows, int K, int tid, int nthreads) {
    const int chunks = K >> 3;
    for (int idx = tid; idx < rows * chunks; idx += nthreads) {
        const int row = idx / chunks, cg = idx - row * chunks;
        const int blk = cg >> 3, c = cg & 7;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (row < valid_rows) v = __ldg(reinterpret_cast<const uint4*>(g + (size_t)row * K) + cg);
        *reinterpret_cast<uint4*>(smem + (size_t)blk * rows * 128 + (size_t)row * 128 + ((c ^ (row & 7)) << 4)) = v;
    }
}

// descriptor of k-step s (16 bf16) for rows [row0, row0 + 64 or N) of a SWIZZLE_128B tile of
// `rows` rows: 64-element K block s / 4 (pitch rows x 128 B), 32 B per k-step inside it
__device__ __forceinline__ uint64_t sw128_desc(uint32_t tile_base, int rows, int row0, int s) {
    return make_smem_desc(tile_base + (uint32_t)(s >> 2) * rows * 128 + (uint32_t)row0 * 128 + (uint32_t)(s & 3) * 32,
                          16, 1024, 1);
}

// Copy a [rows, K] row-major bf16 tile from global memory into the canonical no-swizzle K-major
// layout: 16-byte chunk (row, kc) -> smem[(kc * rows + row) * 16 B].  Rows >= valid_rows are zero.
// Core matrices (8 rows x 16 B) are 128 B apart along M/N (SBO) and rows x 16 B apart along K (LBO).
__device__ __forceinline__ void load_tile_kmajor(uint8_t* smem, const __nv_bfloat16* __restrict__ g, int rows,
                                                 int valid_rows, int K, int tid, int nthreads) {
    const int chunks = K >> 3;   // 8 bf16 per 16-byte chunk
    for (int idx = tid; idx < rows * chunks; idx += nthreads) {
        const int row = idx % rows, kc = idx / rows;   // consecutive threads -> consecutive rows: conflict-free smem
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (row < valid_rows) v = __ldg(reinterpret_cast<const uint4*>(g + (size_t)row * K) + kc);
        *reinterpret_cast<uint4*>(smem + ((size_t)kc * rows + row) * 16) = v;
    }
}

__device__ __forceinline__ uint64_t kmajor_desc(uint32_t tile_base, int rows, int row0, int s) {
    return make_smem_desc(tile_base + (uint32_t)s * 2 * rows * 16 + (uint32_t)row0 * 16, (uint32_t)rows * 16, 128, 0);
}

// ----------------------------------------------------------------------------------------
// Self-test kernel: out[128, 256] = A[128, K] . B[256, K]^T through wgmma.  Two warpgroups, 64
// rows of A each, 256 / NT m64nNTk16 column blocks of B (NT = 128 or 64, the two instructions the
// candidate kernel issues).
// ----------------------------------------------------------------------------------------
constexpr int kDbgM = 128, kDbgN = 256;

template <int NT>
__global__ void __launch_bounds__(256)
tc_gemm_debug_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ B, int K,
                     float* __restrict__ out, int swizzle) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* sA = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms are 1024-B aligned
    uint8_t* sB = sA + (size_t)kDbgM * K * 2;
    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;

    if (swizzle) {
        load_tile_sw128(sA, A, kDbgM, kDbgM, K, tid, blockDim.x);
        load_tile_sw128(sB, B, kDbgN, kDbgN, K, tid, blockDim.x);
    } else {
        load_tile_kmajor(sA, A, kDbgM, kDbgM, K, tid, blockDim.x);
        load_tile_kmajor(sB, B, kDbgN, kDbgN, K, tid, blockDim.x);
    }
    fence_async_smem();
    __syncthreads();
    const uint32_t a0 = smem_u32(sA), b0 = smem_u32(sB);
    for (int nh = 0; nh < kDbgN / NT; ++nh) {
        float d[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) d[i] = 0.0f;
        wgmma_fence();
        for (int s = 0; s < K / kMmaK; ++s) {
            const uint64_t ad = swizzle ? sw128_desc(a0, kDbgM, wg * kWgM, s) : kmajor_desc(a0, kDbgM, wg * kWgM, s);
            const uint64_t bd = swizzle ? sw128_desc(b0, kDbgN, nh * NT, s) : kmajor_desc(b0, kDbgN, nh * NT, s);
            if constexpr (NT == 128) wgmma_m64n128k16(d, ad, bd, s > 0 ? 1u : 0u);
            else wgmma_m64n64k16(d, ad, bd, s > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_keep(d);
        const int r0 = wg * kWgM + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) {
            const int row = r0 + 8 * ((i >> 1) & 1), col = nh * NT + 8 * (i >> 2) + 2 * (t & 3) + (i & 1);
            out[(size_t)row * kDbgN + col] = d[i];
        }
    }
}

}  // namespace tc
}  // namespace nrc

using namespace nrc;

// Test hook: out f32 [128, 256] = A bf16 [128, K] . B bf16 [256, K]^T  (K multiple of 16, <= 256), through
// wgmma m64n128k16 (n_tile 128) or m64n64k16 (n_tile 64).
extern "C" int nrc_tc_gemm_debug_ntile(const void* a_bf16, const void* b_bf16, int32_t k, int32_t swizzle,
                                       int32_t n_tile, float* out, void* stream) {
    NRC_REQUIRE(k >= 16 && k <= 256 && (k % 16) == 0, NRC_E_LIMIT, "k must be a multiple of 16 in [16, 256]");
    NRC_REQUIRE(!swizzle || (k % 64) == 0, NRC_E_LIMIT, "the SWIZZLE_128B layout needs k % 64 == 0");
    NRC_REQUIRE(n_tile == 64 || n_tile == 128, NRC_E_VALUE, "n_tile must be 64 or 128 (got %d)", n_tile);
    const size_t smem = (size_t)(tc::kDbgM + tc::kDbgN) * k * 2 + 1024;
    auto kern = n_tile == 128 ? tc::tc_gemm_debug_kernel<128> : tc::tc_gemm_debug_kernel<64>;
    NRC_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<1, 256, smem, as_stream(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(a_bf16),
                                              reinterpret_cast<const __nv_bfloat16*>(b_bf16), k, out, swizzle);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// The same with the m64n128k16 instruction (the original signature, kept for its callers).
extern "C" int nrc_tc_gemm_debug(const void* a_bf16, const void* b_bf16, int32_t k, int32_t swizzle, float* out,
                                 void* stream) {
    return nrc_tc_gemm_debug_ntile(a_bf16, b_bf16, k, swizzle, 128, out, stream);
}

// =========================================================================================
// Candidate pass + finalisation
// =========================================================================================
namespace nrc {
namespace tc {

// Candidate kernel.  One CTA owns kMU = 128 users and one contiguous range of item tiles.
//   warpgroups 0, 1  consumers: warpgroup g multiplies users [64 g, 64 g + 64) with every item tile
//                    (D/16 wgmma m64nNTk16 from shared memory), stages the 64 x NT fp32 block in
//                    shared memory and filters it: one thread = one user (CH = 2: two threads, one
//                    per half of the tile, each with its own list) -- running threshold, min-heap of
//                    the LQ best approximate scores, merge-walk over the user's train row,
//                    candidate list
//   warp 8           TMA producer (one thread): item tile -> shared memory (SWIZZLE_128B boxes)
// Pipeline: `nst` shared-memory item stages (full_b: the copy engine's bytes; empty_b: one arrive
// per consumer warp once its wgmmas have read the stage).  The two warpgroups run independently,
// so the tensor core works for one while the other filters.
constexpr int kMaxList = 64;           // threshold rank <= 64 (2*top_k for the tie-replay pass)
constexpr int kMU = 2 * kWgM;          // users per CTA
constexpr int kMaxStages = 4;
constexpr int kCandThreads = 2 * 128 + 32;

struct CandArgs {
    const __nv_bfloat16* Ub;   // [num_eval, D] bf16 rows of the users being evaluated (gathered)
    const __nv_bfloat16* Vb;   // [N, D] bf16 item table
    const float* margin;       // [num_eval] 2 * eps_u (see tc_prepare_users_kernel)
    const int32_t* users;      // [num_eval] user ids (train CSR is indexed by user id)
    const int64_t* train_ptr; const int32_t* train_idx;
    int num_eval, N, D;
    int LQ;                    // rank of the running threshold kept per (user, list)
    int lstride;               // shared-memory words per list (odd: conflict-free whatever entry a lane touches)
    int nst;                   // shared-memory item stages
    int seg_tiles;             // item tiles per grid.y segment
    int nslots;                // candidate lists per user = gridDim.y * CH
    int cap;                   // entries per list
    int32_t* cand;             // [num_eval, nslots, cap] candidate item ids, ascending inside a list
    float* cand_val;           // same shape: the approximate (bf16 tensor-core) score of each candidate
    int32_t* cand_cnt;         // [num_eval, nslots] candidates seen (> cap => overflow)
};

// shared-memory words per staged accumulator row: NT + 4 makes the filter's float4 row reads
// (8 users per phase) conflict-free
template <int NT>
__host__ __device__ constexpr int stage_stride() { return NT + 4; }

template <int NT>
size_t cand_smem_bytes(int D, int nst, int CH, int lstride) {
    return 1024 + (size_t)kMU * D * 2 + (size_t)nst * NT * D * 2 + (size_t)kMU * stage_stride<NT>() * 4 +
           (size_t)CH * kMU * lstride * 4;
}

// CH = threads per user in the filter: 1 -> 64 filtering threads per warpgroup, one user each over
// all NT columns; 2 -> all 128, a user is served by two threads (columns [0, NT/2) and [NT/2, NT)),
// each with its OWN threshold list and candidate list (slot), like two item segments interleaved.
template <int NT, int CH>   // items per tile (wgmma N): 128 (dim <= 128) or 64
__global__ void __launch_bounds__(kCandThreads, 1)
tc_candidate_kernel(const CandArgs P, const __grid_constant__ CUtensorMap tmapV) {
    constexpr int kTmaWarp = 8;
    constexpr int SS = stage_stride<NT>();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms are 1024-B aligned
    const int D = P.D;
    const uint32_t stage_bytes = (uint32_t)NT * D * 2;   // one item operand tile
    uint8_t* sA = smem;                                   // [128 x D] bf16, SWIZZLE_128B blocks
    uint8_t* sB = sA + (size_t)kMU * D * 2;               // nst x [NT x D] bf16
    float* sS = reinterpret_cast<float*>(sB + (size_t)P.nst * stage_bytes);   // [128][SS] staged scores
    float* sList = sS + (size_t)kMU * SS;                                       // [CH][128][lstride]
    __shared__ uint64_t full_b[kMaxStages], empty_b[kMaxStages];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row0 = blockIdx.x * kMU;
    const int t_begin = blockIdx.y * P.seg_tiles;                         // first item tile of this CTA
    const int T = min(P.seg_tiles, (P.N + NT - 1) / NT - t_begin);      // its tile count (>= 1)

    load_tile_sw128(sA, P.Ub + (size_t)row0 * D, kMU, max(0, min(kMU, P.num_eval - row0)), D, tid, kCandThreads);
    for (int i = tid; i < CH * kMU * P.lstride; i += kCandThreads) sList[i] = -INFINITY;
    fence_async_smem();
    if (tid == 0) {
        for (int i = 0; i < kMaxStages; ++i) {
            mbar_init(&full_b[i], 1);    // the producer's arrive.expect_tx; the copy engine completes the bytes
            mbar_init(&empty_b[i], 8);   // one arrive per consumer warp after its wgmmas read the stage
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kTmaWarp) {
        // ---------------- producer (one thread): item tiles -> shared memory by TMA ----------------
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmapV)) : "memory");
            const uint32_t b0 = smem_u32(sB);
            int s = 0, ph = 0;
            for (int t = 0; t < T; ++t) {
                mbar_wait(&empty_b[s], ph ^ 1);
                mbar_arrive_expect_tx(&full_b[s], stage_bytes);
                for (int kb = 0; kb < D / 64; ++kb)   // one NT x 64 box per 128-byte K block
                    tma_load_2d(b0 + (uint32_t)s * stage_bytes + (uint32_t)kb * NT * 128, &tmapV, kb * 64,
                                (t_begin + t) * NT, &full_b[s]);
                if (++s == P.nst) { s = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ---------------- consumers: MMA + filter ----------------
    const int g = warp >> 2, wt = tid & 127;                 // warpgroup (user half) and thread inside it
    float* sSg = sS + (size_t)g * kWgM * SS;
    // filter role: user r of this warpgroup, column half ch
    const int r = wt & (kWgM - 1), ch = wt >> 6;
    const bool filters = CH == 2 || ch == 0;
    constexpr int CW = NT / CH;                              // columns per filtering thread and tile
    const int row = row0 + g * kWgM + r;
    const bool live = filters && row < P.num_eval;
    float* lst = sList + ((size_t)ch * kMU + g * kWgM + r) * P.lstride;
    const int slot = blockIdx.y * CH + (CH == 2 ? ch : 0);
    const float margin = live ? P.margin[row] : 0.0f;
    const int u = live ? P.users[row] : 0;
    const int64_t tb = live ? P.train_ptr[u] : 0;
    const int tl = live ? (int)(P.train_ptr[u + 1] - tb) : 0;
    int32_t* my_cand = P.cand + ((size_t)row * P.nslots + slot) * P.cap;
    float* my_val = P.cand_val + ((size_t)row * P.nslots + slot) * P.cap;
    float thr = -INFINITY, thr_m = live ? -INFINITY : INFINITY;   // padding rows never produce candidates
    int cnt = 0;
    // merge-walk over the user's sorted train row: items arrive in ascending order, so the
    // mask test of a candidate is "advance the cursor to >= item, compare" (amortised O(deg))
    int tpos = 0;
    if (live && t_begin > 0) {   // first train item at or after this segment's first item
        int lo = 0, hi = tl;
        const int first = t_begin * NT;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(P.train_idx + tb + mid) < first) lo = mid + 1; else hi = mid;
        }
        tpos = lo;
    }
    int tnext = (tpos < tl) ? __ldg(P.train_idx + tb + tpos) : INT32_MAX;
    int tahead = (tpos + 1 < tl) ? __ldg(P.train_idx + tb + tpos + 1) : INT32_MAX;   // prefetched: advancing never waits on memory

    const uint32_t a_base = smem_u32(sA), b_base = smem_u32(sB);
    const int nks = D / kMmaK;
    const int fr0 = 16 * (wt >> 5) + ((wt & 31) >> 2);     // accumulator fragment: rows fr0, fr0 + 8
    int s = 0, ph = 0;
    for (int t = 0; t < T; ++t) {
        float acc[NT / 2];   // the first k-step overwrites (scale-d = 0)
        mbar_wait(&full_b[s], ph);
        __syncwarp();   // the filter's loops and the wait diverge; wgmma is .sync.aligned
        wgmma_fence();
        const uint32_t bs = b_base + (uint32_t)s * stage_bytes;
#pragma unroll 4
        for (int ks = 0; ks < nks; ++ks) {
            const uint64_t ad = sw128_desc(a_base, kMU, g * kWgM, ks);
            const uint64_t bd = sw128_desc(bs, NT, 0, ks);
            if constexpr (NT == 128) wgmma_m64n128k16(acc, ad, bd, ks > 0 ? 1u : 0u);
            else wgmma_m64n64k16(acc, ad, bd, ks > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_keep(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_b[s]);   // the shared-memory stage may be refilled
        if (++s == P.nst) { s = 0; ph ^= 1; }
        wg_sync(1 + g);                            // the previous tile's filter is done with sSg
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int c = 8 * j + 2 * (wt & 3);
            *reinterpret_cast<float2*>(sSg + (size_t)fr0 * SS + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(sSg + (size_t)(fr0 + 8) * SS + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        wg_sync(1 + g);
        if (!filters) continue;
        const bool tail = (t_begin + t + 1) * NT > P.N;   // only the catalogue's last tile has columns past N
        const float* srow = sSg + (size_t)r * SS;
#pragma unroll 1
        for (int c = ch * CW; c < ch * CW + CW; c += 32) {
            float v[32];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 q = *reinterpret_cast<const float4*>(srow + c + 4 * i);
                v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
            }
            // cheap common case: the chunk maximum does not reach the threshold
            float t16[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) t16[i] = fmaxf(v[2 * i], v[2 * i + 1]);
#pragma unroll
            for (int i = 0; i < 8; ++i) t16[i] = fmaxf(t16[2 * i], t16[2 * i + 1]);
#pragma unroll
            for (int i = 0; i < 4; ++i) t16[i] = fmaxf(t16[2 * i], t16[2 * i + 1]);
            const float mx = fmaxf(fmaxf(t16[0], t16[1]), fmaxf(t16[2], t16[3]));
            unsigned m = 0u;
            if (mx > thr_m) {   // bit i set when column i can still matter for this user
                unsigned m4[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int i = 0; i < 32; ++i) m4[i & 3] |= (v[i] > thr_m ? 1u : 0u) << i;
                m = (m4[0] | m4[1]) | (m4[2] | m4[3]);
            }
            const int item0 = (t_begin + t) * NT + c;
            if (tail && item0 + 32 > P.N) m &= (item0 >= P.N) ? 0u : ((1u << (P.N - item0)) - 1u);
            while (m) {                       // rare: ~LQ ln(N/LQ) times per user in total
                const int i = __ffs(m) - 1;
                m &= m - 1;
                const float x = srow[c + i];
                if (!(x > thr_m)) continue;   // the threshold may have risen inside this chunk
                const int item = item0 + i;
                while (tnext < item) {
                    ++tpos;
                    tnext = tahead;
                    tahead = (tpos + 1 < tl) ? __ldg(P.train_idx + tb + tpos + 1) : INT32_MAX;
                }
                if (tnext == item) continue;  // train item: masked to -inf by the reference
                if (cnt < P.cap) { my_cand[cnt] = item; my_val[cnt] = x; }
                ++cnt;
                if (x > thr) {                // keep the LQ best approximate scores in a min-heap
                    int hpos = 0;             // replace the root (the LQ-th best) and sift down
                    for (;;) {
                        int hc = 2 * hpos + 1;
                        if (hc >= P.LQ) break;
                        float cv = lst[hc];
                        if (hc + 1 < P.LQ) {
                            const float cv2 = lst[hc + 1];
                            if (cv2 < cv) { cv = cv2; ++hc; }
                        }
                        if (!(cv < x)) break;
                        lst[hpos] = cv;
                        hpos = hc;
                    }
                    lst[hpos] = x;
                    thr = lst[0];
                    thr_m = thr - margin;
                }
            }
        }
    }
    if (live) P.cand_cnt[(size_t)row * P.nslots + slot] = cnt;
}

// bf16 copy of the item table + largest row norm (positive floats order like their bit patterns)
__global__ void tc_prepare_items_kernel(const float* __restrict__ V, int64_t N, int D, __nv_bfloat16* __restrict__ Vb,
                                        unsigned int* __restrict__ vmax_bits) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    float best = 0.0f;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < N; i += warps) {
        float sq = 0.0f;
        for (int k = lane; k < D; k += 32) {
            const float x = V[i * D + k];
            Vb[i * D + k] = __float2bfloat16_rn(x);
            sq = fmaf(x, x, sq);
        }
        sq = warp_sum(sq);
        best = fmaxf(best, sqrtf(sq));
    }
    if (lane == 0) atomicMax(vmax_bits, __float_as_uint(best));
}

// bf16 rows of the evaluated users + their candidate margin
//   bf16 keeps 8 significant bits, so round-to-nearest has unit roundoff 2^-8 per FACTOR:
//   u^_k v^_k = u_k v_k (1+a)(1+b), |a|,|b| <= 2^-8  =>  |u^.v^ - u.v| <= (2^-7 + 2^-16) sum|u_k v_k|
//   <= (2^-7 + 2^-16) |u| |v| (Cauchy-Schwarz).  The fp32 accumulation of the tensor core (truncating
//   adder, d <= 192 terms) and the fp32 FMA chain of the exact score add < 2^-11 |u| |v| together.
//   eps = (2^-7 + 2^-11) * |u| * max_i |v_i| * 1.001 (norms are fp32-rounded), margin = 2 * eps:
//   an item's approximate score and the order statistic it is compared with each move by <= eps.
//   The wgmma accumulation term is measured by tests/test_gpu_tc_eval.py (adversarial k = 256 operands:
//   <= 2^-20 sum|u_k v_k|), and subnormal products by tests/test_gpu_tc_candidates.py (within eps).
__global__ void tc_prepare_users_kernel(const float* __restrict__ U, const int32_t* __restrict__ users, int num_eval,
                                        int D, const unsigned int* __restrict__ vmax_bits,
                                        __nv_bfloat16* __restrict__ Ub, float* __restrict__ margin) {
    const int lane = threadIdx.x & 31;
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= num_eval) return;
    const float* u = U + (size_t)users[row] * D;
    float sq = 0.0f;
    for (int k = lane; k < D; k += 32) {
        const float x = u[k];
        Ub[(size_t)row * D + k] = __float2bfloat16_rn(x);
        sq = fmaf(x, x, sq);
    }
    sq = warp_sum(sq);
    if (lane == 0) {
        const float vmax = __uint_as_float(*vmax_bits);
        margin[row] = 2.0f * (0.0078125f + 0.00048828125f) * sqrtf(sq) * vmax * 1.001f;
    }
}

}  // namespace tc
}  // namespace nrc

#include "tc_eval.cuh"

namespace nrc {
namespace tc {

// library-owned workspaces, grown on demand (never inside a stream capture)
struct Arena {
    void* p = nullptr;
    size_t bytes = 0;
    int reserve(size_t need) {
        if (need <= bytes) return NRC_OK;
        if (p) NRC_CUDA_CHECK(cudaFree(p));
        p = nullptr; bytes = 0;
        NRC_CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        return NRC_OK;
    }
};
static Arena g_items;          // bf16 item table + max row norm
static Arena g_pass[2];        // per pass: bf16 user rows, margins, candidate lists and counts
static const __nv_bfloat16* g_vb = nullptr;
static unsigned int* g_vmax = nullptr;
static int g_items_n = 0, g_items_d = 0;
static cudaEvent_t g_ev[2] = {nullptr, nullptr};   // around the last main-pass tc_candidate_kernel launch
static double g_last_flops = 0.0;

static size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

// The bf16 copy + max row norm are reused across calls while the caller vouches that the table has
// not changed: nrc_eval_tc_items_version(v != 0) keys the cache on (pointer, shape, v); version 0
// (default) converts on every call.
static int g_ch_pref = 1;       // filter threads per user: 1 (default) or 2 (nrc_eval_tc_epilogue_warps)
static int g_force_segments = 0;   // item segments per pass: 0 = heuristic, g >= 1 = min(g, tiles) (nrc_eval_tc_force_segments)
static uint64_t g_items_version = 0, g_cached_version = 0;
static const float* g_cached_ptr = nullptr;

int prepare_items(const float* V, int D, int N, cudaStream_t st) {
    NRC_REQUIRE(D % 64 == 0 && D >= 64 && D <= 256, NRC_E_LIMIT,
                "the tensor-core pass needs dim in {64, 128, 192, 256} (got %d)", D);
    if (g_items_version != 0 && g_cached_version == g_items_version && g_cached_ptr == V && g_items_n == N &&
        g_items_d == D && g_vb != nullptr)
        return NRC_OK;
    const size_t o_vmax = up256((size_t)N * D * 2);
    int rc = g_items.reserve(o_vmax + 256);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(g_items.p);
    __nv_bfloat16* Vb = reinterpret_cast<__nv_bfloat16*>(ws);
    g_vmax = reinterpret_cast<unsigned int*>(ws + o_vmax);
    NRC_CUDA_CHECK(cudaMemsetAsync(g_vmax, 0, 4, st));
    tc_prepare_items_kernel<<<sm_count() * 8, 256, 0, st>>>(V, N, D, Vb, g_vmax);
    NRC_CUDA_CHECK(cudaGetLastError());
    g_vb = Vb; g_items_n = N; g_items_d = D;
    g_cached_ptr = V; g_cached_version = g_items_version;
    return NRC_OK;
}

int run_pass(int pass, const float* U, const int32_t* users, int num_rows, const int64_t* train_ptr,
             const int32_t* train_idx, int LQ, int cap, CandLists* out, cudaStream_t st) {
    NRC_REQUIRE(pass == 0 || pass == 1, NRC_E_VALUE, "pass must be 0 or 1");
    NRC_REQUIRE(g_vb != nullptr, NRC_E_VALUE, "prepare_items has not run");
    NRC_REQUIRE(LQ >= 1 && LQ <= kMaxList, NRC_E_LIMIT, "threshold rank %d outside [1, %d]", LQ, kMaxList);
    const int D = g_items_d, N = g_items_n;
    const int row_tiles = (num_rows + kMU - 1) / kMU;
    // Tile width: 128 items (wgmma N) while two stages of them fit beside the staged scores; 64 for dim 192.
    const int lstride = (LQ <= 32) ? 33 : 65;
    const int CH = (g_ch_pref == 2 && pass == 0) ? 2 : 1;   // the replay pass needs lists in ascending item order
    const int kNT = (D <= 128) ? 128 : 64;
    const size_t fixed = (kNT == 128 ? cand_smem_bytes<128>(D, 0, CH, lstride) : cand_smem_bytes<64>(D, 0, CH, lstride));
    const size_t smem_max = 227 * 1024 - 1024;   // opt-in limit minus the static barriers, rounded
    const size_t budget = fixed < smem_max ? smem_max - fixed : 0;
    const int T = (N + kNT - 1) / kNT;
    // Item segments (grid.y): with few user tiles, split the catalogue so that every SM has a CTA.
    // Each segment restarts its threshold (still a lower bound of the true one), which costs a few
    // more candidates; pick the split with the fewest waves per unit of work, at most 8 unless a
    // single wave needs more (16 at most; 48 in the replay pass), and never segments shorter
    // than 4096 items.
    int G = 1;
    {
        const int sms = sm_count();
        const int few = (pass == 1) ? 48 : 16;   // the replay pass re-scores its lists with a whole CTA per user
        const int gmax = (row_tiles * 8 < sms) ? ((sms / row_tiles < few) ? sms / row_tiles : few) : 8;
        double best = 1e30;
        const int min_tiles = 4096 / kNT;
        for (int g = 1; g <= gmax && g * min_tiles <= (T > min_tiles ? T : min_tiles); ++g) {
            const int ctas = row_tiles * g;
            const double cost = (double)((ctas + sms - 1) / sms) / g * (1.0 + 0.02 * (g - 1));
            if (cost < best - 1e-9) { best = cost; G = g; }
        }
    }
    if (g_force_segments > 0) G = g_force_segments < T ? g_force_segments : T;   // test hook
    const int seg_tiles = (T + G - 1) / G;
    G = (T + seg_tiles - 1) / seg_tiles;           // no empty segment
    const int nslots = G * CH;
    int nst = (int)(budget / ((size_t)kNT * D * 2));
    if (nst > kMaxStages) nst = kMaxStages;
    NRC_REQUIRE(nst >= 2, NRC_E_LIMIT, "dim %d with threshold rank %d does not fit the tensor-core pass", D, LQ);
    const size_t rows_pad = (size_t)row_tiles * kMU;
    const size_t o_ub = 0;
    const size_t o_margin = o_ub + up256(rows_pad * D * 2);
    const size_t o_cnt = o_margin + up256(rows_pad * 4);
    const size_t o_cand = o_cnt + up256(rows_pad * nslots * 4);
    const size_t o_scr = o_cand + up256(rows_pad * (size_t)nslots * cap * 4);
    const size_t total = o_scr + up256(rows_pad * (size_t)nslots * cap * 4);
    int rc = g_pass[pass].reserve(total);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(g_pass[pass].p);
    __nv_bfloat16* Ub = reinterpret_cast<__nv_bfloat16*>(ws + o_ub);
    float* margin = reinterpret_cast<float*>(ws + o_margin);
    int32_t* cnt = reinterpret_cast<int32_t*>(ws + o_cnt);
    int32_t* cd = reinterpret_cast<int32_t*>(ws + o_cand);
    tc_prepare_users_kernel<<<(num_rows * 32 + 255) / 256, 256, 0, st>>>(U, users, num_rows, D, g_vmax, Ub, margin);
    NRC_CUDA_CHECK(cudaGetLastError());

    CandArgs P{Ub, g_vb, margin, users, train_ptr, train_idx, num_rows, N, D,
               LQ, lstride, nst, seg_tiles, nslots, cap, cd, reinterpret_cast<float*>(ws + o_scr), cnt};
    CUtensorMap tmapV;
    {   // bf16 item table [N, D] row-major; box = kNT items x 64 k (one 128-byte swizzle span)
        static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
        if (!encode) {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult q;
            NRC_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
            NRC_REQUIRE(fn != nullptr && q == cudaDriverEntryPointSuccess, NRC_E_CUDA,
                        "the driver does not export cuTensorMapEncodeTiled");
            encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
        }
        const cuuint64_t gdim[2] = {(cuuint64_t)D, (cuuint64_t)N};
        const cuuint64_t gstride[1] = {(cuuint64_t)D * 2};
        const cuuint32_t box[2] = {64u, (cuuint32_t)kNT};
        const cuuint32_t estr[2] = {1u, 1u};
        const CUresult cr = encode(&tmapV, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)g_vb, gdim, gstride, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        NRC_REQUIRE(cr == CUDA_SUCCESS, NRC_E_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
    }
    const size_t smem = fixed + (size_t)nst * kNT * D * 2;
    static bool attr_done = false;
    if (!attr_done) {
        NRC_CUDA_CHECK(cudaFuncSetAttribute(tc_candidate_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_max));
        NRC_CUDA_CHECK(cudaFuncSetAttribute(tc_candidate_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_max));
        NRC_CUDA_CHECK(cudaFuncSetAttribute(tc_candidate_kernel<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_max));
        NRC_CUDA_CHECK(cudaFuncSetAttribute(tc_candidate_kernel<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem_max));
        attr_done = true;
    }
    const dim3 grid(row_tiles, G);
    if (pass == 0) {
        if (!g_ev[0]) {
            NRC_CUDA_CHECK(cudaEventCreate(&g_ev[0]));
            NRC_CUDA_CHECK(cudaEventCreate(&g_ev[1]));
        }
        NRC_CUDA_CHECK(cudaEventRecord(g_ev[0], st));
    }
    if (CH == 2) {
        if (kNT == 128) tc_candidate_kernel<128, 2><<<grid, kCandThreads, smem, st>>>(P, tmapV);
        else tc_candidate_kernel<64, 2><<<grid, kCandThreads, smem, st>>>(P, tmapV);
    } else {
        if (kNT == 128) tc_candidate_kernel<128, 1><<<grid, kCandThreads, smem, st>>>(P, tmapV);
        else tc_candidate_kernel<64, 1><<<grid, kCandThreads, smem, st>>>(P, tmapV);
    }
    NRC_CUDA_CHECK(cudaGetLastError());
    if (pass == 0) {
        NRC_CUDA_CHECK(cudaEventRecord(g_ev[1], st));
        g_last_flops = 2.0 * (double)num_rows * (double)N * (double)D;
    }
    out->cand = cd;
    out->scratch = reinterpret_cast<float*>(ws + o_scr);
    out->margin = margin;
    out->cnt = cnt;
    out->nslots = nslots;
    out->cap = cap;
    out->seg_items = seg_tiles * kNT;
    return NRC_OK;
}

}  // namespace tc
}  // namespace nrc

// Evaluations of one fixed model in several calls (user batches) share the bf16 item table: set a
// non-zero version before the first call and keep it while the table is unchanged; any other value
// (or 0 = never cache) makes the next call convert again.
extern "C" int nrc_eval_tc_items_version(uint64_t version) {
    nrc::tc::g_items_version = version;
    return NRC_OK;
}

// Filter layout of the main pass's candidate kernel: 8 (default) = one thread per user, 16 = every user
// is served by two threads, one per half of each item tile, each with its own threshold and candidate list.
extern "C" int nrc_eval_tc_epilogue_warps(int32_t warps) {
    NRC_REQUIRE(warps == 8 || warps == 16, NRC_E_VALUE, "epilogue warps must be 8 or 16 (got %d)", warps);
    nrc::tc::g_ch_pref = warps / 8;
    return NRC_OK;
}

// Test hook: item segments (grid.y) of both candidate passes.  0 = the occupancy heuristic of run_pass;
// g >= 1 = min(g, item tiles) segments (then the same "no empty segment" recount).
extern "C" int nrc_eval_tc_force_segments(int32_t g) {
    NRC_REQUIRE(g >= 0, NRC_E_VALUE, "segment count must be >= 0 (got %d)", g);
    nrc::tc::g_force_segments = g;
    return NRC_OK;
}

// Test hook: one candidate pass exactly as nrc_eval_mf_tc runs it (prepare_items + run_pass: the same CH rule,
// the same forced or heuristic segment count), with the lists copied out.  cand / cand_val [n, nslots, cap],
// cnt [n, nslots], margin [n] are device buffers sized for max_slots lists per row; *nslots and *seg_items
// are host outputs.
extern "C" int nrc_eval_tc_debug_candidates(int32_t pass, const float* user_table, const float* item_table,
                                            int32_t dim, int32_t num_items, const int32_t* users, int32_t n,
                                            const int64_t* train_indptr, const int32_t* train_indices, int32_t lq,
                                            int32_t cap, int32_t max_slots, int32_t* cand, float* cand_val,
                                            int32_t* cnt, float* margin, int32_t* nslots, int32_t* seg_items,
                                            void* stream) {
    NRC_REQUIRE(nslots != nullptr && seg_items != nullptr, NRC_E_VALUE, "NULL output");
    NRC_REQUIRE(n > 0 && cap > 0 && num_items > 0, NRC_E_VALUE, "bad shape");
    cudaStream_t st = as_stream(stream);
    int rc = nrc::tc::prepare_items(item_table, dim, num_items, st);
    if (rc) return rc;
    nrc::tc::CandLists c;
    rc = nrc::tc::run_pass(pass, user_table, users, n, train_indptr, train_indices, lq, cap, &c, st);
    if (rc) return rc;
    *nslots = c.nslots;
    *seg_items = c.seg_items;
    NRC_REQUIRE(c.nslots <= max_slots, NRC_E_LIMIT, "the pass uses %d lists per row (> max_slots %d)", c.nslots,
                max_slots);
    const size_t lists = (size_t)n * c.nslots;
    NRC_CUDA_CHECK(cudaMemcpyAsync(cand, c.cand, lists * cap * 4, cudaMemcpyDeviceToDevice, st));
    NRC_CUDA_CHECK(cudaMemcpyAsync(cand_val, c.scratch, lists * cap * 4, cudaMemcpyDeviceToDevice, st));
    NRC_CUDA_CHECK(cudaMemcpyAsync(cnt, c.cnt, lists * 4, cudaMemcpyDeviceToDevice, st));
    NRC_CUDA_CHECK(cudaMemcpyAsync(margin, c.margin, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    return NRC_OK;
}

// Duration (CUDA events on the launching stream) and algorithmic flops (2 * users * items * dim)
// of the last candidate-kernel launch; waits for that launch to finish.
extern "C" int nrc_eval_tc_last_launch(float* kernel_ms, double* flops) {
    NRC_REQUIRE(kernel_ms != nullptr && flops != nullptr, NRC_E_VALUE, "NULL output");
    NRC_REQUIRE(nrc::tc::g_ev[0] != nullptr, NRC_E_VALUE, "nrc_eval_mf_tc has not run yet");
    NRC_CUDA_CHECK(cudaEventSynchronize(nrc::tc::g_ev[1]));
    NRC_CUDA_CHECK(cudaEventElapsedTime(kernel_ms, nrc::tc::g_ev[0], nrc::tc::g_ev[1]));
    *flops = nrc::tc::g_last_flops;
    return NRC_OK;
}
