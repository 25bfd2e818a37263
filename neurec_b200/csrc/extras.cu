// SURVEY.md 8(f) ranks 3-4: the other embedding-BPR consumers of the fused triplet path and the
// data-side helpers around them.
//
// Replaces (reference paths):
//   model/general_recommender/APR.py:92-118     _create_adversarial: delta = l2_normalize(rows) * eps
//   model/social_recommender/SBPR.py:66-92      _create_inference / _create_loss (user, item, social item, negative, s_uk)
//   model/social_recommender/SBPR.py:103-149    train_model's batch loop + _get_pairwise_all_data (per-epoch sampling)
//   data/sampler.py:216-354 (+ :42-68)          TimeOrder*Sampler: the recent-items window travels with the shuffled sample
//   data/dataset.py:288-296, util/tool.py:56-65 interactions -> CSR with ascending rows (device build)
//
// SBPR's epoch is, like the MF epoch (epoch.cuh), a pure function of (train CSR, social-item CSR, trust CSR,
// seed, epoch): position p of the shuffled epoch -> positive `perm(p)` -> its user's social item (uniform over the
// user's social-item row, with replacement: np.random.choice, SBPR.py:139), its negative (uniform over the
// items outside train(u) + social(u): randint_choice with exclusion, SBPR.py:135-137) and
// s_uk = 1 + #{trusted f : social item in train(f)} (SBPR.py:141-145).
#include "common.cuh"
#include "epoch.cuh"
#include "extras.cuh"
#include "learner.cuh"
#include "optim.cuh"
#include "philox.cuh"

namespace nrc {

// ---------------------------------------------------------------------------------------------
// APR: tf.nn.l2_normalize(x, 1) * eps  ==  (x * rsqrt(max(sum(x^2), 1e-12))) * eps, one warp per row
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
l2_normalize_rows_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t rows, int dim, float scale) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += (int64_t)gridDim.x * wpb) {
        const float* __restrict__ p = x + r * dim;
        float ss = 0.0f;
        for (int k = lane; k < dim; k += kWarp) ss = fmaf(p[k], p[k], ss);
        ss = warp_sum(ss);
        const float inv = rsqrtf(fmaxf(ss, 1e-12f));
        for (int k = lane; k < dim; k += kWarp) out[r * dim + k] = (p[k] * inv) * scale;
    }
}

// ---------------------------------------------------------------------------------------------
// int32 row gather: out[p, :] = src[index[p] % src_rows, :]   (the recent-items window of TimeOrder samplers:
// the pointwise layout repeats the positives neg_num + 1 times, sampler.py:259-260, hence the modulo)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gather_rows_i32_kernel(const int32_t* __restrict__ src, int64_t src_rows, int width, const int64_t* __restrict__ index,
                       int64_t n, int32_t* __restrict__ out) {
    const int64_t total = n * width;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = e / width;
        const int c = (int)(e - p * width);
        out[e] = __ldg(src + (__ldg(index + p) % src_rows) * width + c);
    }
}

// ---------------------------------------------------------------------------------------------
// SBPR epoch
// ---------------------------------------------------------------------------------------------
struct SbprSpec {
    const int64_t* tptr; const int32_t* tidx;     // train CSR, ascending rows
    const int64_t* sptr; const int32_t* sidx;     // social items of every user (items of trusted users outside the user's own row), ascending
    const int64_t* fptr; const int32_t* fidx;     // trust CSR: social_matrix[u].indices
    const int32_t* users; const int32_t* pos;     // flattened positives of the users that have social items
    int64_t n;
    int32_t num_items;
    uint64_t seed, stream_id;
    Feistel perm;
};

constexpr uint64_t kSocialStream = 0x534F4349414C0000ull;   // 'SOCIAL': the social-item draw's own stream

__device__ __forceinline__ void sbpr_sample(const SbprSpec& S, int64_t p, int32_t& u, int32_t& i, int32_t& k,
                                            int32_t& j, float& suk) {
    const int64_t idx = feistel_perm(S.perm, p);
    u = __ldg(S.users + idx);
    i = __ldg(S.pos + idx);
    const int64_t tb = __ldg(S.tptr + u), tdeg = __ldg(S.tptr + u + 1) - tb;
    const int64_t sb = __ldg(S.sptr + u), sdeg = __ldg(S.sptr + u + 1) - sb;
    // np.random.choice(socialItemsList, size=pos_len): uniform with replacement over the user's social items
    k = __ldg(S.sidx + sb + philox_candidate((uint64_t)idx, 0, S.seed ^ kSocialStream, S.stream_id, (int32_t)sdeg));
    // randint_choice(num_items, pos_len, replace=True, exclusion=social + pos)
    for (uint32_t a = 0;; ++a) {
        const int32_t c = philox_candidate((uint64_t)idx, a, S.seed, S.stream_id, S.num_items);
        if (!sorted_contains(S.tidx + tb, tdeg, c) && !sorted_contains(S.sidx + sb, sdeg, c)) { j = c; break; }
    }
    // socialWeight = sum over trusted users of [k in train(f)] + 1
    int cnt = 1;
    const int64_t fb = __ldg(S.fptr + u), fe = __ldg(S.fptr + u + 1);
    for (int64_t q = fb; q < fe; ++q) {
        const int32_t f = __ldg(S.fidx + q);
        const int64_t b = __ldg(S.tptr + f);
        cnt += sorted_contains(S.tidx + b, __ldg(S.tptr + f + 1) - b, k) ? 1 : 0;
    }
    suk = (float)cnt;
}

__global__ void __launch_bounds__(256)
sbpr_epoch_build_kernel(const SbprSpec S, int64_t first, int64_t count, int32_t* __restrict__ ou, int32_t* __restrict__ oi,
                        int32_t* __restrict__ ok, int32_t* __restrict__ oj, float* __restrict__ os) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < count; e += (int64_t)gridDim.x * blockDim.x) {
        int32_t u, i, k, j;
        float s;
        sbpr_sample(S, first + e, u, i, k, j, s);
        ou[e] = u; oi[e] = i; ok[e] = k; oj[e] = j; os[e] = s;
    }
}

// One warp per (user, positive, social, negative, s_uk) sample.  SBPR.py:66-92:
//   x_* = <p, q_*> + b_*;  r1 = (x_i - x_k) / s;  r2 = x_k - x_j
//   loss = l(r1) + l(r2) + reg * l2_loss(p, q_k, q_i, q_j, b_i, b_k, b_j)
// Row gradients go to the dense accumulators (duplicates sum = IndexedSlices de-duplication); the three
// embedding_lookups of the user row contribute one summed gradient.
__global__ void __launch_bounds__(256)
sbpr_grad_kernel(const float* __restrict__ U, const float* __restrict__ V, const float* __restrict__ B, int D,
                 const int32_t* __restrict__ users, const int32_t* __restrict__ pos, const int32_t* __restrict__ soc,
                 const int32_t* __restrict__ neg, const float* __restrict__ suk, int64_t batch, int loss_kind, float reg,
                 float* __restrict__ gU, float* __restrict__ gV, float* __restrict__ gB, int32_t* __restrict__ tU,
                 int32_t* __restrict__ tV, int32_t stamp, float* __restrict__ loss) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    float loss_acc = 0.0f;
    for (int64_t b = blockIdx.x * wpb + (threadIdx.x >> 5); b < batch; b += (int64_t)gridDim.x * wpb) {
        const int u = users[b], i = pos[b], k = soc[b], j = neg[b];
        const float s = suk[b];
        const float* __restrict__ pu = U + (size_t)u * D;
        const float* __restrict__ qi = V + (size_t)i * D;
        const float* __restrict__ qk = V + (size_t)k * D;
        const float* __restrict__ qj = V + (size_t)j * D;
        float di = 0.f, dk = 0.f, dj = 0.f, sq = 0.f;
        for (int t = lane; t < D; t += kWarp) {
            const float a = pu[t], vi = qi[t], vk = qk[t], vj = qj[t];
            di = fmaf(a, vi, di); dk = fmaf(a, vk, dk); dj = fmaf(a, vj, dj);
            sq += a * a + vi * vi + vk * vk + vj * vj;
        }
        di = warp_sum(di); dk = warp_sum(dk); dj = warp_sum(dj);
        const float bi = B[i], bk = B[k], bj = B[j];
        const float xi = di + bi, xk = dk + bk, xj = dj + bj;
        float l1, g1, l2, g2;
        pairwise_loss_grad(loss_kind, (xi - xk) / s, l1, g1);
        pairwise_loss_grad(loss_kind, xk - xj, l2, g2);
        float l = l1 + l2;
        if (reg != 0.0f) l += reg * 0.5f * (warp_sum(sq) + bi * bi + bk * bk + bj * bj);
        loss_acc += l;
        const float ci = g1 / s, ck = g2 - ci, cj = -g2;      // dl/dx_i, dl/dx_k, dl/dx_j
        float* gu = gU + (size_t)u * D;
        float* gi = gV + (size_t)i * D;
        float* gk = gV + (size_t)k * D;
        float* gj = gV + (size_t)j * D;
        for (int t = lane; t < D; t += kWarp) {
            const float a = pu[t], vi = qi[t], vk = qk[t], vj = qj[t];
            atomicAdd(gu + t, ci * vi + ck * vk + cj * vj + reg * a);
            atomicAdd(gi + t, ci * a + reg * vi);
            atomicAdd(gk + t, ck * a + reg * vk);
            atomicAdd(gj + t, cj * a + reg * vj);
        }
        if (lane == 0) {
            atomicAdd(gB + i, ci + reg * bi);
            atomicAdd(gB + k, ck + reg * bk);
            atomicAdd(gB + j, cj + reg * bj);
            tU[u] = stamp; tV[i] = stamp; tV[k] = stamp; tV[j] = stamp;
        }
    }
    if (lane == 0 && loss) atomicAdd(loss, loss_acc);
}

// ---------------------------------------------------------------------------------------------
// interactions (COO, any order, duplicates allowed) -> CSR with ascending, duplicate-free rows
//   1 count per row (RED), 2 exclusive scan (host-launched single CTA; rows <= 2^31), 3 scatter, 4 per-row
//   insertion sort + de-duplication (warp per row), 5 compaction by a second scan.
// Small helper kernels only; the sort is per row because rows are short (median 52 on ml-100k) and a row is
// the unit every consumer binary-searches.
// ---------------------------------------------------------------------------------------------
__global__ void coo_count_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ cols, int64_t nnz, int32_t num_rows,
                                 int32_t num_cols, int64_t* __restrict__ cnt, int32_t* __restrict__ bad) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = rows[e], c = cols[e];
        if (r < 0 || r >= num_rows || c < 0 || c >= num_cols) { *bad = 1; continue; }
        atomicAdd(reinterpret_cast<unsigned long long*>(cnt + r + 1), 1ull);
    }
}

// in-place inclusive scan of ptr[1..n] (ptr[0] = 0) by ONE 1024-thread CTA; chunked, carries between chunks
__global__ void __launch_bounds__(1024) scan_i64_kernel(int64_t* __restrict__ ptr, int64_t n) {
    __shared__ int64_t warp_tot[32];
    __shared__ int64_t carry_s;
    if (threadIdx.x == 0) { carry_s = 0; ptr[0] = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t e = base + threadIdx.x;
        int64_t v = (e < n) ? ptr[e + 1] : 0;
        for (int o = 1; o < 32; o <<= 1) { const int64_t t = __shfl_up_sync(kFull, v, o); if (lane >= o) v += t; }
        if (lane == 31) warp_tot[w] = v;
        __syncthreads();
        if (w == 0) {
            int64_t t = warp_tot[lane];
            for (int o = 1; o < 32; o <<= 1) { const int64_t x = __shfl_up_sync(kFull, t, o); if (lane >= o) t += x; }
            warp_tot[lane] = t;
        }
        __syncthreads();
        const int64_t off = carry_s + (w ? warp_tot[w - 1] : 0);
        if (e < n) ptr[e + 1] = v + off;
        __syncthreads();
        if (threadIdx.x == 0) carry_s += warp_tot[31];
        __syncthreads();
    }
}

__global__ void coo_scatter_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ cols, int64_t nnz, int32_t num_rows,
                                   int32_t num_cols, const int64_t* __restrict__ ptr, int64_t* __restrict__ cursor,
                                   int32_t* __restrict__ out) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = rows[e], c = cols[e];
        if (r < 0 || r >= num_rows || c < 0 || c >= num_cols) continue;      // flagged by the counting pass
        const int64_t slot = (int64_t)atomicAdd(reinterpret_cast<unsigned long long*>(cursor + r), 1ull);
        out[ptr[r] + slot] = cols[e];
    }
}

// one warp per row, rank sort: the output position of an element is the number of smaller elements, ties broken by
// position -- O(deg^2 / 32) per row, deterministic whatever order the scatter pass left, and rows are short.
__global__ void __launch_bounds__(256)
csr_sort_rows_kernel(const int64_t* __restrict__ ptr, int32_t num_rows, const int32_t* __restrict__ in, int32_t* __restrict__ out,
                     int64_t* __restrict__ uniq) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < num_rows; r += (int64_t)gridDim.x * wpb) {
        const int64_t b = ptr[r], deg = ptr[r + 1] - b;
        // rank sort: out position of element e = #{x < v} + #{x == v at an earlier position}
        for (int64_t e = lane; e < deg; e += kWarp) {
            const int32_t v = in[b + e];
            int64_t rank = 0;
            for (int64_t q = 0; q < deg; ++q) {
                const int32_t x = __ldg(in + b + q);
                rank += (x < v) || (x == v && q < e);
            }
            out[b + rank] = v;
        }
        __syncwarp();
        // count distinct values (row is sorted now): the compaction pass reads this
        int64_t u = 0;
        for (int64_t e = lane; e < deg; e += kWarp) u += (e == 0) || (out[b + e] != out[b + e - 1]);
        for (int o = 16; o > 0; o >>= 1) u += __shfl_xor_sync(kFull, u, o);
        if (lane == 0) uniq[r + 1] = u;
    }
}

__global__ void __launch_bounds__(256)
csr_compact_rows_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ new_ptr, int32_t num_rows,
                        const int32_t* __restrict__ sorted, int32_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < num_rows; r += (int64_t)gridDim.x * wpb) {
        const int64_t b = ptr[r], deg = ptr[r + 1] - b;
        int64_t w = new_ptr[r];
        for (int64_t base = 0; base < deg; base += kWarp) {
            const int64_t e = base + lane;
            const bool keep = e < deg && (e == 0 || sorted[b + e] != sorted[b + e - 1]);
            const unsigned m = __ballot_sync(kFull, keep);
            if (keep) out[w + __popc(m & ((1u << lane) - 1u))] = sorted[b + e];
            w += __popc(m);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Per-user train / test split (data/utils.py:59-106): order every user's interactions by key -- the interaction time
// (by_time=True) or a counter-based random word (by_time=False: DataFrame.sample(frac=1), a uniformly random order) --
// ties by position in the input, and send the first cut(n_u) to the train set:
//   ratio  cut = ceil(ratio * n_u)                        (split_by_ratio, :59-80)
//   loo    cut = n_u if n_u <= 3 else n_u - 1             (split_by_loo, :83-106)
// One warp per user, rank by counting (rows are short).
// ---------------------------------------------------------------------------------------------
__global__ void index_scatter_kernel(const int32_t* __restrict__ rows, int64_t n, int32_t num_rows, const int64_t* __restrict__ ptr,
                                     int64_t* __restrict__ cursor, int32_t* __restrict__ out) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = rows[e];
        if (r < 0 || r >= num_rows) continue;
        const int64_t slot = (int64_t)atomicAdd(reinterpret_cast<unsigned long long*>(cursor + r), 1ull);
        out[ptr[r] + slot] = (int32_t)e;
    }
}

__global__ void coo_count_rows_kernel(const int32_t* __restrict__ rows, int64_t n, int32_t num_rows, int64_t* __restrict__ cnt,
                                      int32_t* __restrict__ bad) {
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = rows[e];
        if (r < 0 || r >= num_rows) { *bad = 1; continue; }
        atomicAdd(reinterpret_cast<unsigned long long*>(cnt + r + 1), 1ull);
    }
}

constexpr uint64_t kSplitStream = 0x53504C4954000000ull;    // 'SPLIT'

__global__ void __launch_bounds__(256)
split_rank_kernel(const int64_t* __restrict__ ptr, int32_t num_users, const int32_t* __restrict__ seg, const int64_t* __restrict__ keys,
                  int mode, double ratio, uint64_t seed, int32_t* __restrict__ is_train) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t u = blockIdx.x * wpb + (threadIdx.x >> 5); u < num_users; u += (int64_t)gridDim.x * wpb) {
        const int64_t b = ptr[u], n = ptr[u + 1] - b;
        const int64_t cut = mode == 0 ? (int64_t)ceil(ratio * (double)n) : (n <= 3 ? n : n - 1);
        for (int64_t e = lane; e < n; e += kWarp) {
            const int32_t me = seg[b + e];
            // keys are compared as unsigned 64-bit words: times are shifted by 2^63 to keep their signed order
            const uint64_t ke = keys ? ((uint64_t)keys[me] ^ 0x8000000000000000ull) : philox_word((uint64_t)me, 0, seed, kSplitStream);
            int64_t rank = 0;
            for (int64_t q = 0; q < n; ++q) {
                const int32_t other = __ldg(seg + b + q);
                const uint64_t kq = keys ? ((uint64_t)__ldg(keys + other) ^ 0x8000000000000000ull)
                                         : philox_word((uint64_t)other, 0, seed, kSplitStream);
                rank += (kq < ke) || (kq == ke && other < me);
            }
            is_train[me] = rank < cut ? 1 : 0;
        }
    }
}

// users_list of _generate_positive_items (data/sampler.py:24-39) from the CSR row pointers: out[e] = row of entry e.
// One warp per row (rows of a train CSR are short; a 700-entry row is 22 strides).
__global__ void __launch_bounds__(256)
csr_row_ids_kernel(const int64_t* __restrict__ ptr, int64_t num_rows, int32_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t wpb = blockDim.x >> 5;
    for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < num_rows; r += (int64_t)gridDim.x * wpb) {
        const int64_t b = __ldg(ptr + r), e = __ldg(ptr + r + 1);
        for (int64_t q = b + lane; q < e; q += kWarp) out[q] = (int32_t)r;
    }
}

static unsigned grid_for(int64_t work_items, int per_block) {
    int64_t blocks = (work_items + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

// 1 when grid_for capped the grid, so a thread (per_block 256) or warp (per_block 8) takes more than one item
static int grid_capped(int64_t work_items, int per_block) {
    return (work_items + per_block - 1) / per_block > (int64_t)sm_count() * 8 ? 1 : 0;
}

// Host record of the most recent launch of each kernel group, for nrc_extras_last_routes (see the header).
static struct ExtrasRoutes {
    int32_t r[kExKernels][kExFields];
    ExtrasRoutes() { for (auto& k : r) for (auto& f : k) f = -1; }
} g_extras_routes;

void extras_route(int kernel, int64_t grid, int capped, int64_t row_grid, int row_capped, int64_t scan_chunks,
                  int replace) {
    int32_t* r = g_extras_routes.r[kernel];
    r[kExGrid] = (int32_t)grid; r[kExCapped] = capped; r[kExRowGrid] = (int32_t)row_grid; r[kExRowCapped] = row_capped;
    r[kExScanChunks] = (int32_t)scan_chunks; r[kExReplace] = replace;
}

static int sbpr_spec_init(SbprSpec& S, const int64_t* tptr, const int32_t* tidx, const int64_t* sptr, const int32_t* sidx,
                          const int64_t* fptr, const int32_t* fidx, const int32_t* users, const int32_t* pos, int64_t n,
                          int32_t num_items, int32_t max_excluded, int32_t shuffle, uint64_t seed, uint64_t epoch) {
    NRC_REQUIRE(num_items > 0 && n >= 0, NRC_E_VALUE, "num_items must be positive, n >= 0");
    // random_choice.pyx:32-33
    NRC_REQUIRE(max_excluded < num_items, NRC_E_VALUE, "The number of 'exclusion' is greater than 'high'.");
    S.tptr = tptr; S.tidx = tidx; S.sptr = sptr; S.sidx = sidx; S.fptr = fptr; S.fidx = fidx;
    S.users = users; S.pos = pos; S.n = n; S.num_items = num_items; S.seed = seed; S.stream_id = epoch;
    return feistel_init(S.perm, n, shuffle, seed, epoch);
}

}  // namespace nrc

using namespace nrc;

extern "C" int nrc_l2_normalize_rows(const float* x, int64_t rows, int32_t dim, float scale, float* out, void* stream) {
    NRC_REQUIRE(rows >= 0 && dim > 0, NRC_E_VALUE, "bad table shape");
    if (rows == 0) return NRC_OK;
    NRC_REQUIRE(x && out, NRC_E_VALUE, "NULL table");
    extras_route(kExL2Normalize, grid_for(rows, 8), grid_capped(rows, 8));
    l2_normalize_rows_kernel<<<grid_for(rows, 8), 256, 0, as_stream(stream)>>>(x, out, rows, dim, scale);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_gather_rows_i32(const int32_t* src, int64_t src_rows, int32_t width, const int64_t* index, int64_t n,
                                   int32_t* out, void* stream) {
    NRC_REQUIRE(src_rows > 0 && width > 0 && n >= 0, NRC_E_VALUE, "bad gather shape");
    if (n == 0) return NRC_OK;
    extras_route(kExGatherRows, grid_for(n * width, 256), grid_capped(n * width, 256));
    gather_rows_i32_kernel<<<grid_for(n * width, 256), 256, 0, as_stream(stream)>>>(src, src_rows, width, index, n, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_sbpr_epoch_build(const int64_t* train_indptr, const int32_t* train_indices, const int64_t* social_indptr,
                                    const int32_t* social_indices, const int64_t* trust_indptr, const int32_t* trust_indices,
                                    const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos, int32_t num_items,
                                    int32_t max_excluded, int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t first,
                                    int64_t count, int32_t* out_users, int32_t* out_pos, int32_t* out_social,
                                    int32_t* out_neg, float* out_suk, void* stream) {
    SbprSpec S;
    const int rc = sbpr_spec_init(S, train_indptr, train_indices, social_indptr, social_indices, trust_indptr, trust_indices,
                                  pos_users, pos_items, n_pos, num_items, max_excluded, shuffle, seed, epoch);
    if (rc) return rc;
    NRC_REQUIRE(first >= 0 && count >= 0 && first + count <= n_pos, NRC_E_VALUE, "window [%lld, %lld) outside the epoch of %lld samples",
                (long long)first, (long long)(first + count), (long long)n_pos);
    if (count == 0) return NRC_OK;
    extras_route(kExSbprEpochBuild, grid_for(count, 256), grid_capped(count, 256));
    sbpr_epoch_build_kernel<<<grid_for(count, 256), 256, 0, as_stream(stream)>>>(S, first, count, out_users, out_pos, out_social,
                                                                                  out_neg, out_suk);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

extern "C" int nrc_sbpr_grad(const float* user_table, const float* item_table, const float* item_bias, int32_t dim,
                             const int32_t* users, const int32_t* pos_items, const int32_t* social_items,
                             const int32_t* neg_items, const float* suk, int64_t batch, int32_t loss_kind, float reg,
                             float* grad_user, float* grad_item, float* grad_bias, int32_t* touched_user,
                             int32_t* touched_item, int32_t stamp, float* loss, void* stream) {
    NRC_REQUIRE(dim > 0 && batch >= 0, NRC_E_VALUE, "dim > 0 and batch >= 0 required");
    // learner.py:27-28
    NRC_REQUIRE(loss_kind >= NRC_LOSS_BPR && loss_kind <= NRC_LOSS_SQUARE, NRC_E_VALUE, "please choose a suitable loss function");
    if (batch == 0) return NRC_OK;
    extras_route(kExSbprGrad, grid_for(batch, 8), grid_capped(batch, 8));
    sbpr_grad_kernel<<<grid_for(batch, 8), 256, 0, as_stream(stream)>>>(user_table, item_table, item_bias, dim, users, pos_items,
                                                                         social_items, neg_items, suk, batch, loss_kind, reg,
                                                                         grad_user, grad_item, grad_bias, touched_user,
                                                                         touched_item, stamp, loss);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// SBPR.train_model's batch loop (SBPR.py:111-121) over an epoch already built on the device: per batch the gradient
// kernel + ONE optimizer launch over the three variables (bias = a [num_items, 1] table sharing the items' stamps).
extern "C" int nrc_sbpr_train_epoch(float* user_table, float* item_table, float* item_bias, int32_t num_users,
                                    int32_t num_items, int32_t dim, const int32_t* users, const int32_t* pos_items,
                                    const int32_t* social_items, const int32_t* neg_items, const float* suk, int64_t n,
                                    int32_t batch_size, int32_t loss_kind, float reg, int32_t opt_kind,
                                    const float* lr_t_host, const float* hyper_host, float* grad_user, float* grad_item,
                                    float* grad_bias, int32_t* touched_user, int32_t* touched_item, float* slot0_user,
                                    float* slot1_user, float* slot0_item, float* slot1_item, float* slot0_bias,
                                    float* slot1_bias, int32_t first_stamp, float* step_loss, void* stream) {
    NRC_REQUIRE(batch_size > 0, NRC_E_VALUE, "batch_size should be a positive integeral value");
    NRC_REQUIRE(n >= 0 && dim > 0, NRC_E_VALUE, "n >= 0 and dim > 0 required");
    cudaStream_t st = as_stream(stream);
    const int64_t steps = (n + batch_size - 1) / batch_size;
    if (steps == 0) return NRC_OK;
    NRC_CUDA_CHECK(cudaMemsetAsync(step_loss, 0, (size_t)steps * sizeof(float), st));
    float hyper[4] = {hyper_host[0], hyper_host[1], hyper_host[2], hyper_host[3]};
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t off = s * batch_size;
        const int64_t bs = (n - off < batch_size) ? (n - off) : batch_size;
        const int32_t stamp = first_stamp + (int32_t)s;
        int rc = nrc_sbpr_grad(user_table, item_table, item_bias, dim, users + off, pos_items + off, social_items + off,
                               neg_items + off, suk + off, bs, loss_kind, reg, grad_user, grad_item, grad_bias, touched_user,
                               touched_item, stamp, step_loss + s, stream);
        if (rc) return rc;
        if (opt_kind == NRC_OPT_ADAM) hyper[0] = lr_t_host[s];
        OptLaunch L;
        rc = opt_launch_init(L, opt_kind, hyper);
        if (rc) return rc;
        opt_launch_add(L, user_table, grad_user, slot0_user, slot1_user, touched_user, num_users, dim, 0);
        opt_launch_add(L, item_table, grad_item, slot0_item, slot1_item, touched_item, num_items, dim, 0);
        opt_launch_add(L, item_bias, grad_bias, slot0_bias, slot1_bias, touched_item, num_items, 1, 0);
        rc = opt_launch_run(L, stamp, st);
        if (rc) return rc;
    }
    return NRC_OK;
}

// interactions -> CSR (rows ascending and duplicate-free).  out_indices needs room for nnz entries; scratch: work_i64
// [2 * (num_rows + 1)], work_i32 [2 * nnz].  out_indptr[num_rows] (device) is the number of distinct interactions;
// *bad_flag (device i32) becomes 1 when an id was outside [0, num_rows) x [0, num_cols) (those entries are dropped).
extern "C" int nrc_csr_from_coo(const int32_t* rows, const int32_t* cols, int64_t nnz, int32_t num_rows, int32_t num_cols,
                                int64_t* out_indptr, int32_t* out_indices, int64_t* work_i64, int32_t* work_i32,
                                int32_t* bad_flag, void* stream) {
    NRC_REQUIRE(num_rows > 0 && num_cols > 0 && nnz >= 0, NRC_E_VALUE, "num_rows > 0, num_cols > 0 and nnz >= 0 required");
    cudaStream_t st = as_stream(stream);
    int64_t* raw_ptr = work_i64;                       // [num_rows + 1] row pointers with duplicates
    int64_t* cursor = work_i64 + (num_rows + 1);       // [num_rows + 1] scatter cursors (only the first num_rows used)
    int32_t* scattered = work_i32;                     // [nnz]
    int32_t* sorted = work_i32 + nnz;                  // [nnz]
    NRC_CUDA_CHECK(cudaMemsetAsync(raw_ptr, 0, (size_t)(num_rows + 1) * 8, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(cursor, 0, (size_t)(num_rows + 1) * 8, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(out_indptr, 0, (size_t)(num_rows + 1) * 8, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(bad_flag, 0, 4, st));
    extras_route(kExCsrFromCoo, nnz ? grid_for(nnz, 256) : 0, nnz ? grid_capped(nnz, 256) : 0, grid_for(num_rows, 8),
                 grid_capped(num_rows, 8), ((int64_t)num_rows + 1023) / 1024);
    if (nnz) coo_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(rows, cols, nnz, num_rows, num_cols, raw_ptr, bad_flag);
    scan_i64_kernel<<<1, 1024, 0, st>>>(raw_ptr, num_rows);
    if (nnz) coo_scatter_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(rows, cols, nnz, num_rows, num_cols, raw_ptr, cursor, scattered);
    csr_sort_rows_kernel<<<grid_for(num_rows, 8), 256, 0, st>>>(raw_ptr, num_rows, scattered, sorted, out_indptr);
    scan_i64_kernel<<<1, 1024, 0, st>>>(out_indptr, num_rows);
    csr_compact_rows_kernel<<<grid_for(num_rows, 8), 256, 0, st>>>(raw_ptr, out_indptr, num_rows, sorted, out_indices);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// data/utils.py:59-106 on the device.  users i32 [n] (dense ids); keys i64 [n] = interaction times (by_time=True) or NULL
// (by_time=False: counter-based random order keyed by `seed`); mode 0 = ratio, 1 = leave-one-out.  is_train i32 [n]
// receives 1 / 0 per interaction (interactions of out-of-range users are left untouched and *bad_flag is set).
// Scratch: work_i64 [2 * (num_users + 1)], work_i32 [n].
extern "C" int nrc_split_interactions(const int32_t* users, const int64_t* keys, int64_t n, int32_t num_users, int32_t mode,
                                      double ratio, uint64_t seed, int32_t* is_train, int64_t* work_i64, int32_t* work_i32,
                                      int32_t* bad_flag, void* stream) {
    NRC_REQUIRE(num_users > 0 && n >= 0, NRC_E_VALUE, "num_users > 0 and n >= 0 required");
    NRC_REQUIRE(mode == 0 || mode == 1, NRC_E_VALUE, "There is not splitter '%d'", mode);       // dataset.py:160-161
    NRC_REQUIRE(mode == 1 || (ratio >= 0.0 && ratio <= 1.0), NRC_E_VALUE, "ratio %f outside [0, 1]", ratio);
    cudaStream_t st = as_stream(stream);
    int64_t* ptr = work_i64;
    int64_t* cursor = work_i64 + (num_users + 1);
    NRC_CUDA_CHECK(cudaMemsetAsync(ptr, 0, (size_t)(num_users + 1) * 8, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(cursor, 0, (size_t)(num_users + 1) * 8, st));
    NRC_CUDA_CHECK(cudaMemsetAsync(bad_flag, 0, 4, st));
    if (n == 0) return NRC_OK;
    extras_route(kExSplit, grid_for(n, 256), grid_capped(n, 256), grid_for(num_users, 8), grid_capped(num_users, 8),
                 ((int64_t)num_users + 1023) / 1024);
    coo_count_rows_kernel<<<grid_for(n, 256), 256, 0, st>>>(users, n, num_users, ptr, bad_flag);
    scan_i64_kernel<<<1, 1024, 0, st>>>(ptr, num_users);
    index_scatter_kernel<<<grid_for(n, 256), 256, 0, st>>>(users, n, num_users, ptr, cursor, work_i32);
    split_rank_kernel<<<grid_for(num_users, 8), 256, 0, st>>>(ptr, num_users, work_i32, keys, mode, ratio, seed, is_train);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// The flattened positives' users (data/sampler.py:24-39 `users_list`) expanded on the device from the CSR row pointers,
// so that only (indptr, indices) have to cross PCIe.  out i32 [indptr[num_rows]].
extern "C" int nrc_csr_row_ids(const int64_t* indptr, int64_t num_rows, int32_t* out, void* stream) {
    NRC_REQUIRE(num_rows >= 0, NRC_E_VALUE, "num_rows >= 0 required");
    if (num_rows == 0) return NRC_OK;
    extras_route(kExCsrRowIds, grid_for(num_rows, 8), grid_capped(num_rows, 8));
    csr_row_ids_kernel<<<grid_for(num_rows, 8), 256, 0, as_stream(stream)>>>(indptr, num_rows, out);
    NRC_CUDA_CHECK(cudaGetLastError());
    return NRC_OK;
}

// Host bookkeeping of the routes the most recent data-side, sampler and LightGCN-gradient launches took (see the
// header); no device work.
extern "C" int nrc_extras_last_routes(int32_t* out) {
    NRC_REQUIRE(out != nullptr, NRC_E_VALUE, "out is NULL");
    for (int k = 0; k < kExKernels; ++k)
        for (int f = 0; f < kExFields; ++f) out[k * kExFields + f] = g_extras_routes.r[k][f];
    return NRC_OK;
}
