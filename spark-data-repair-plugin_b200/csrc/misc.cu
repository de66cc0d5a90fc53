// Kernels behind delphi.misc (RepairMiscApi.scala): k-means assignment over dictionary codes,
// error maps, NULL injection and table flattening.
//
// dr_kmeans_assign never sees a row's bag-of-q-grams vector.  With P_c = B_c mu^T (one row per
// dictionary slot of column c, slot 0 = NULL, one column per centre) the squared distance to centre j
// is ||x||^2 + ||mu_j||^2 - 2 sum_c P_c[slot_c(r)][j], so the argmin reads K codes per row and gathers
// K rows of P.  Each lane takes 4 consecutive rows per 128-bit load of a column (the k_scan_hist
// pattern), the dot products accumulate over the columns in table order from 0.0 with __dadd_rn and
// the score is mu_sq[j] - 2 dot, ties to the lower j: the host reproduces every label bit for bit.
#include "common.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kTileRows = 128;   // rows per warp: 4 per lane
constexpr int kJ = 8;            // centres per accumulation pass (4 rows x 8 doubles in registers)
constexpr size_t kSmemBudget = 200 * 1024;

struct AssignParams {
    const int32_t* cols[DR_MAX_COLS];
    uint32_t dom[DR_MAX_COLS];     // slot clamp: slot = min(code + 1, dom)
    int32_t p_off[DR_MAX_COLS];    // row of P holding column c's slot 0
    int n_cols;
    int n_centres;
    int64_t n_rows;
    int64_t p_rows;
    const double* P;               // [p_rows][n_centres]
    const double* mu_sq;           // [n_centres]
    const int32_t* split;          // [n_labels] or nullptr
    int32_t n_labels;
    int32_t* labels;
    int vec;                       // every column and `labels` 16-byte aligned
};

__device__ __forceinline__ int4 load4(const int32_t* __restrict__ a, int64_t r0, int64_t n, bool vec, bool stream) {
    if (vec && r0 + 4 <= n) {
        const int4* p = reinterpret_cast<const int4*>(a + r0);
        return stream ? __ldcs(p) : __ldg(p);
    }
    int4 v;
    v.x = r0 < n ? a[r0] : -1;
    v.y = r0 + 1 < n ? a[r0 + 1] : -1;
    v.z = r0 + 2 < n ? a[r0 + 2] : -1;
    v.w = r0 + 3 < n ? a[r0 + 3] : -1;
    return v;
}

__device__ __forceinline__ unsigned slot_of(int code, unsigned dom) { return min((unsigned)(code + 1), dom); }

__device__ __forceinline__ double score(double mu, double dot) { return __dsub_rn(mu, __dmul_rn(2.0, dot)); }

template <bool kSmem>
__device__ __forceinline__ const double* stage_p(const AssignParams& p, double* sm, const double** mu) {
    if (!kSmem) {
        *mu = p.mu_sq;
        return p.P;
    }
    const int64_t np = p.p_rows * p.n_centres;
    for (int64_t i = threadIdx.x; i < np; i += kThreads) sm[i] = __ldg(p.P + i);
    for (int i = threadIdx.x; i < p.n_centres; i += kThreads) sm[np + i] = __ldg(p.mu_sq + i);
    __syncthreads();
    *mu = sm + np;
    return sm;
}

// Plain Lloyd assignment: every row takes the nearest of all n_centres centres.
template <bool kSmem>
__global__ void __launch_bounds__(kThreads) k_kmeans_assign(const __grid_constant__ AssignParams p) {
    extern __shared__ double sm[];
    const double* mu;
    const double* P = stage_p<kSmem>(p, sm, &mu);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nc = p.n_centres;
    const bool single_pass = nc <= kJ;
    const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
    for (int64_t t = (int64_t)blockIdx.x * kWarps + warp; t < n_tiles; t += (int64_t)gridDim.x * kWarps) {
        const int64_t r0 = t * kTileRows + lane * 4;
        if (r0 >= p.n_rows) continue;
        double best[4];
        int bj[4] = {0, 0, 0, 0};
        for (int j0 = 0; j0 < nc; j0 += kJ) {
            double acc[4][kJ];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < kJ; ++j) acc[i][j] = 0.0;
            for (int c = 0; c < p.n_cols; ++c) {
                const int4 q = load4(p.cols[c], r0, p.n_rows, p.vec, single_pass);
                const unsigned dom = p.dom[c];
                const double* base = P + (int64_t)p.p_off[c] * nc + j0;
                const double* row[4] = {base + (int64_t)slot_of(q.x, dom) * nc, base + (int64_t)slot_of(q.y, dom) * nc,
                                        base + (int64_t)slot_of(q.z, dom) * nc, base + (int64_t)slot_of(q.w, dom) * nc};
#pragma unroll
                for (int j = 0; j < kJ; ++j)
                    if (j0 + j < nc) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[i][j] = __dadd_rn(acc[i][j], row[i][j]);
                    }
            }
#pragma unroll
            for (int j = 0; j < kJ; ++j)
                if (j0 + j < nc) {
                    const double m = mu[j0 + j];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const double s = score(m, acc[i][j]);
                        if (j0 + j == 0 || s < best[i]) { best[i] = s; bj[i] = j0 + j; }
                    }
                }
        }
        if (p.vec && r0 + 4 <= p.n_rows) {
            *reinterpret_cast<int4*>(p.labels + r0) = make_int4(bj[0], bj[1], bj[2], bj[3]);
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (r0 + i < p.n_rows) p.labels[r0 + i] = bj[i];
        }
    }
}

// Bisecting step: a row labelled L with split[L] = s >= 0 takes the nearer of centres s and s + 1;
// every other row keeps its label.
template <bool kSmem>
__global__ void __launch_bounds__(kThreads) k_kmeans_assign_split(const __grid_constant__ AssignParams p) {
    extern __shared__ double sm[];
    const double* mu;
    const double* P = stage_p<kSmem>(p, sm, &mu);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nc = p.n_centres;
    const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
    for (int64_t t = (int64_t)blockIdx.x * kWarps + warp; t < n_tiles; t += (int64_t)gridDim.x * kWarps) {
        const int64_t r0 = t * kTileRows + lane * 4;
        if (r0 >= p.n_rows) continue;
        const int4 l4 = load4(p.labels, r0, p.n_rows, p.vec, false);
        const int lab[4] = {l4.x, l4.y, l4.z, l4.w};
        int s[4];
        bool any = false;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            s[i] = (r0 + i < p.n_rows && lab[i] >= 0 && lab[i] < p.n_labels) ? __ldg(p.split + lab[i]) : -1;
            if (s[i] < 0 || s[i] + 1 >= nc) s[i] = -1;
            any |= s[i] >= 0;
        }
        if (!any) continue;
        double a0[4] = {0.0, 0.0, 0.0, 0.0}, a1[4] = {0.0, 0.0, 0.0, 0.0};
        for (int c = 0; c < p.n_cols; ++c) {
            const int4 q = load4(p.cols[c], r0, p.n_rows, p.vec, true);
            const int code[4] = {q.x, q.y, q.z, q.w};
            const unsigned dom = p.dom[c];
            const double* base = P + (int64_t)p.p_off[c] * nc;
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (s[i] >= 0) {
                    const double* row = base + (int64_t)slot_of(code[i], dom) * nc + s[i];
                    a0[i] = __dadd_rn(a0[i], row[0]);
                    a1[i] = __dadd_rn(a1[i], row[1]);
                }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (s[i] >= 0) p.labels[r0 + i] = score(mu[s[i] + 1], a1[i]) < score(mu[s[i]], a0[i]) ? s[i] + 1 : s[i];
    }
}

// ---- error map: one '*' / '-' byte per (row, attribute), row-major -------------------------------
__global__ void k_error_map(const uint32_t* const* __restrict__ bm, int K, int64_t n_rows, uint8_t* __restrict__ out) {
    const int64_t total = n_rows * K;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
    for (int64_t o = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; o < total; o += stride) {
        int64_t r = o / K;
        int c = (int)(o - r * K);
        uint32_t w = 0;
        const int m = total - o < 4 ? (int)(total - o) : 4;
        for (int b = 0; b < m; ++b) {
            const uint32_t* col = bm[c];
            const bool err = col != nullptr && ((__ldg(col + (r >> 5)) >> (r & 31)) & 1u);
            w |= (uint32_t)(err ? '*' : '-') << (8 * b);
            if (++c == K) { c = 0; ++r; }
        }
        if (m == 4 && ((uintptr_t)(out + o) & 3) == 0) {
            *reinterpret_cast<uint32_t*>(out + o) = w;
        } else {
            for (int b = 0; b < m; ++b) out[o + b] = (uint8_t)(w >> (8 * b));
        }
    }
}

// ---- NULL injection: keep = valid && u > ratio, u = top 53 bits of splitmix64 over (key, row) ------
__device__ __forceinline__ uint64_t splitmix(uint64_t row, uint64_t key) {
    uint64_t z = row * 0x9E3779B97F4A7C15ull + key;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void k_null_bits(const uint32_t* __restrict__ valid, int64_t bit_offset, int64_t n_rows, int64_t row_base,
                            uint64_t key, double ratio, uint32_t* __restrict__ out) {
    const int64_t n_words = (bit_offset + n_rows + 31) >> 5;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
        uint32_t keep = 0;
        for (int b = 0; b < 32; ++b) {
            const int64_t r = (w << 5) + b - bit_offset;
            if (r < 0 || r >= n_rows) continue;
            const uint64_t u = splitmix((uint64_t)(row_base + r), key) >> 11;
            if ((double)u * 0x1p-53 > ratio) keep |= 1u << b;
        }
        out[w] = valid != nullptr ? (keep & __ldg(valid + w)) : keep;
    }
}

// ---- flatten: cell (r, c) -> output row r * K + c ----------------------------------------------
__global__ void k_flatten(const int32_t* const* __restrict__ cols, const int64_t* __restrict__ base, int K,
                          int64_t n_rows, const int64_t* __restrict__ ids, int32_t* __restrict__ out_codes,
                          uint32_t* __restrict__ out_valid, int64_t* __restrict__ out_ids) {
    const int64_t total = n_rows * K;
    const int64_t padded = (total + 31) & ~(int64_t)31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;   // a multiple of 32: warps stay word-aligned
    for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < padded; o += stride) {
        bool ok = false;
        if (o < total) {
            const int64_t r = o / K;
            const int c = (int)(o - r * K);
            const int code = __ldg(cols[c] + r);
            ok = code >= 0;
            out_codes[o] = ok ? (int32_t)(code + base[c]) : 0;
            out_ids[o] = ids != nullptr ? __ldg(ids + r) : r;
        }
        const unsigned w = __ballot_sync(0xffffffffu, ok);
        if ((threadIdx.x & 31) == 0) out_valid[o >> 5] = w;
    }
}

// ---- (label, value) counts in global memory: the centre-update counts of a column whose table is
// too large for dr_cooc's shared-memory tables.  Only labels in [lo, hi) are counted.
__global__ void k_label_counts(const int32_t* __restrict__ labels, const int32_t* __restrict__ col, uint32_t dom,
                               int64_t n_rows, int32_t lo, int32_t hi, unsigned long long* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
        const int l = __ldcs(labels + r);
        if (l < lo || l >= hi) continue;
        const unsigned s = slot_of(__ldcs(col + r), dom);
        atomicAdd(out + (int64_t)(l - lo) * (dom + 1) + s, 1ull);
    }
}

// Copies a small host table (column pointers, bases) into the context scratch buffer.
int to_scratch(dr_ctx* ctx, const void* host, size_t bytes, cudaStream_t st, void** dev) {
    int rc = dr_ensure_scratch(ctx, bytes);
    if (rc) return rc;
    // the previous user of the scratch buffer may still be reading it
    DR_CUDA(ctx, cudaStreamSynchronize(st));
    DR_CUDA(ctx, cudaMemcpyAsync(ctx->scratch, host, bytes, cudaMemcpyHostToDevice, st));
    DR_CUDA(ctx, cudaStreamSynchronize(st));
    *dev = ctx->scratch;
    return DR_OK;
}

}  // namespace

extern "C" {

int dr_kmeans_assign(dr_ctx* ctx, const int32_t* const* cols, const int32_t* dom, const int64_t* p_off, int n_cols,
                     int64_t n_rows, const double* P, int64_t p_rows, const double* mu_sq, int32_t n_centres,
                     const int32_t* split, int32_t n_labels, int32_t* labels, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, cols && dom && p_off && P && mu_sq && labels, "null pointer");
    DR_REQUIRE(ctx, n_cols >= 1 && n_cols <= DR_MAX_COLS, "n_cols must be in [1, 64]");
    DR_REQUIRE(ctx, n_rows >= 0 && n_rows < (int64_t)INT32_MAX, "n_rows must be < 2^31 per shard");
    DR_REQUIRE(ctx, n_centres >= 1, "n_centres must be positive");
    DR_REQUIRE(ctx, split == nullptr || n_labels >= 1, "split needs n_labels >= 1");
    DR_REQUIRE(ctx, p_rows >= 1 && p_rows * (int64_t)n_centres < ((int64_t)1 << 40), "bad P size");
    AssignParams p;
    memset(&p, 0, sizeof(p));
    bool vec = ((uintptr_t)labels & 15) == 0;
    for (int c = 0; c < n_cols; ++c) {
        DR_REQUIRE(ctx, cols[c] != nullptr, "null column pointer");
        DR_REQUIRE(ctx, dom[c] >= 0, "negative domain size");
        DR_REQUIRE(ctx, p_off[c] >= 0 && p_off[c] + dom[c] + 1 <= p_rows && p_off[c] < INT32_MAX,
                   "P rows of a column out of range");
        p.cols[c] = cols[c];
        p.dom[c] = (uint32_t)dom[c];
        p.p_off[c] = (int32_t)p_off[c];
        vec = vec && ((uintptr_t)cols[c] & 15) == 0;
    }
    if (n_rows == 0) return DR_OK;
    p.n_cols = n_cols;
    p.n_centres = n_centres;
    p.n_rows = n_rows;
    p.p_rows = p_rows;
    p.P = P;
    p.mu_sq = mu_sq;
    p.split = split;
    p.n_labels = n_labels;
    p.labels = labels;
    p.vec = vec;
    cudaStream_t st = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t smem = (size_t)(p_rows * n_centres + n_centres) * sizeof(double);
    const bool in_smem = smem <= kSmemBudget;
    const int64_t n_tiles = (n_rows + kTileRows - 1) / kTileRows;
    const int per_sm = in_smem ? (int)(220 * 1024 / (smem + 1024) < 4 ? 220 * 1024 / (smem + 1024) : 4) : 4;
    const int grid = dr_grid_for(ctx, n_tiles, kWarps, per_sm < 1 ? 1 : per_sm);
    auto launch = [&](auto kernel, size_t bytes) -> int {
        if (bytes > 48 * 1024) DR_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        kernel<<<grid, kThreads, bytes, st>>>(p);
        DR_LAUNCHED(ctx);
        return DR_OK;
    };
    if (split == nullptr) return in_smem ? launch(k_kmeans_assign<true>, smem) : launch(k_kmeans_assign<false>, 0);
    return in_smem ? launch(k_kmeans_assign_split<true>, smem) : launch(k_kmeans_assign_split<false>, 0);
}

int dr_label_counts(dr_ctx* ctx, const int32_t* labels, const int32_t* col, int32_t dom, int64_t n_rows,
                    int32_t lab_lo, int32_t lab_hi, int64_t* out, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, labels && col && out, "null pointer");
    DR_REQUIRE(ctx, dom >= 0 && dom < INT32_MAX, "bad domain size");
    DR_REQUIRE(ctx, lab_lo >= 0 && lab_hi > lab_lo, "label range must be non-empty");
    DR_REQUIRE(ctx, n_rows >= 0 && n_rows < (int64_t)INT32_MAX, "n_rows must be < 2^31 per shard");
    if (n_rows == 0) return DR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaSetDevice(ctx->device));
    const int threads = 256;
    const int grid = dr_grid_for(ctx, n_rows, threads, 8);
    k_label_counts<<<grid, threads, 0, st>>>(labels, col, (uint32_t)dom, n_rows, lab_lo, lab_hi,
                                             reinterpret_cast<unsigned long long*>(out));
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_error_map(dr_ctx* ctx, const uint32_t* const* bitmaps, int n_attrs, int64_t n_rows, uint8_t* out,
                 void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, bitmaps && out, "null pointer");
    DR_REQUIRE(ctx, n_attrs >= 1 && n_attrs <= (1 << 20), "n_attrs must be in [1, 2^20]");
    DR_REQUIRE(ctx, n_rows >= 0 && n_rows < (int64_t)INT32_MAX, "n_rows must be < 2^31");
    if (n_rows == 0) return DR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaSetDevice(ctx->device));
    void* d = nullptr;
    int rc = to_scratch(ctx, bitmaps, sizeof(void*) * (size_t)n_attrs, st, &d);
    if (rc) return rc;
    const int threads = 256;
    const int grid = dr_grid_for(ctx, (n_rows * n_attrs + 3) / 4, threads, 8);
    k_error_map<<<grid, threads, 0, st>>>((const uint32_t* const*)d, n_attrs, n_rows, out);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_null_bits(dr_ctx* ctx, const uint32_t* valid, int64_t bit_offset, int64_t n_rows, int64_t row_base,
                 uint64_t key, double ratio, uint32_t* out, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, out != nullptr, "null pointer");
    DR_REQUIRE(ctx, n_rows >= 0 && bit_offset >= 0 && row_base >= 0, "negative size or offset");
    DR_REQUIRE(ctx, ratio == ratio, "ratio is NaN");
    if (n_rows == 0) return DR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaSetDevice(ctx->device));
    const int threads = 256;
    const int grid = dr_grid_for(ctx, (bit_offset + n_rows + 31) / 32, threads, 8);
    k_null_bits<<<grid, threads, 0, st>>>(valid, bit_offset, n_rows, row_base, key, ratio, out);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_flatten(dr_ctx* ctx, const int32_t* const* cols, const int64_t* base, int n_cols, int64_t n_rows,
               const int64_t* row_ids, int32_t* out_codes, uint32_t* out_valid, int64_t* out_ids, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, cols && base && out_codes && out_valid && out_ids, "null pointer");
    DR_REQUIRE(ctx, n_cols >= 1 && n_cols <= (1 << 20), "n_cols must be in [1, 2^20]");
    DR_REQUIRE(ctx, n_rows >= 0 && n_rows < (int64_t)INT32_MAX, "n_rows must be < 2^31");
    for (int c = 0; c < n_cols; ++c) {
        DR_REQUIRE(ctx, cols[c] != nullptr, "null column pointer");
        DR_REQUIRE(ctx, base[c] >= 0 && base[c] < INT32_MAX, "column base out of range");
    }
    if (n_rows == 0) return DR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t bytes = sizeof(void*) * (size_t)n_cols + sizeof(int64_t) * (size_t)n_cols;
    void* host = malloc(bytes);
    if (!host) return dr_fail(ctx, DR_ERR_INVALID, "out of host memory");
    memcpy(host, cols, sizeof(void*) * (size_t)n_cols);
    memcpy((char*)host + sizeof(void*) * (size_t)n_cols, base, sizeof(int64_t) * (size_t)n_cols);
    void* d = nullptr;
    int rc = to_scratch(ctx, host, bytes, st, &d);
    free(host);
    if (rc) return rc;
    const int threads = 256;
    const int grid = dr_grid_for(ctx, n_rows * n_cols, threads, 8);
    k_flatten<<<grid, threads, 0, st>>>((const int32_t* const*)d,
                                        (const int64_t*)((char*)d + sizeof(void*) * (size_t)n_cols), n_cols, n_rows,
                                        row_ids, out_codes, out_valid, out_ids);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

}  // extern "C"
