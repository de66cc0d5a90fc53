// LOFOutlierErrorDetector: scikit-learn's LocalOutlierFactor(novelty=False) with its defaults, fitted on
// one continuous column, computed over the column's sorted dictionary instead of per row.
//
// In one dimension the k nearest neighbours of a point are a contiguous run of the sorted order, so every
// copy of a value has the same neighbour multiset and hence the same kdist / lrd / lof.  The input is the
// D distinct values u[0] < ... < u[D-1] with their multiplicities cnt[i] (>= 1); entry i's neighbours are
// cnt[i] - 1 copies of itself, then whole runs taken outward, nearest first (an equal-distance tie takes
// the smaller value first), the last run possibly partial.  A window therefore spans at most k entries on
// each side, and lof_i depends only on entries within 3k of i.
//
// Three grid-stride passes, each staging a tile of entries plus a halo of k on each side in shared memory
// (every window read is a shared-memory load):
//   1. kdist_i = distance of the run that completes k
//   2. lrd_i   = 1 / (S_i / k + 1e-10),   S_i = sum_j m_ij * max(d(i,j), kdist_j)
//   3. lof_i   = L_i / k,                 L_i = sum_j m_ij * (lrd_j / lrd_i);   verdict = lof_i > 1.5
// Sums run over the window in ascending value order; every float operation is an explicit __d*_rn, so
// the results are bit-identical to the NumPy restatement in oracle/lof.py.
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;
constexpr int kTile = kThreads * kPerThread;   // entries per tile
constexpr int kMaxK = 64;
constexpr int kStage = kTile + 2 * kMaxK;

struct Window {
    int64_t lo, hi;          // first / last entry of the window (lo <= i <= hi)
    int64_t m_lo, m_hi;      // multiplicity taken from entry lo / hi (when it is not i itself)
    int64_t m_self;          // copies of entry i among its own neighbours
    double kdist;
};

// su / sc: staged entries, local index = global index - base
__device__ __forceinline__ Window lof_window(const double* su, const long long* sc, int64_t base, int64_t e,
                                             int64_t D, int k) {
    Window w;
    const long long ci = sc[e - base];
    long long m_self = ci - 1 < (long long)k ? ci - 1 : (long long)k;
    if (m_self < 0) m_self = 0;
    long long rem = (long long)k - m_self;
    w.lo = w.hi = e;
    w.m_lo = w.m_hi = 0;
    w.m_self = m_self;
    w.kdist = 0.0;
    const double ue = su[e - base];
    int64_t l = e - 1, r = e + 1;
    while (rem > 0) {
        // (l >= e - k, r <= e + k always hold for counts >= 1; the bounds keep reads inside the halo anyway)
        const bool has_l = l >= 0 && l >= e - k;
        const bool has_r = r < D && r <= e + k;
        if (!has_l && !has_r) break;
        const double dl = has_l ? __dsub_rn(ue, su[l - base]) : 0.0;
        const double dr = has_r ? __dsub_rn(su[r - base], ue) : 0.0;
        if (has_l && (!has_r || dl <= dr)) {
            const long long c = sc[l - base];
            const long long m = c < rem ? c : rem;
            rem -= m;
            w.kdist = dl;
            w.lo = l;
            w.m_lo = m;
            --l;
        } else {
            const long long c = sc[r - base];
            const long long m = c < rem ? c : rem;
            rem -= m;
            w.kdist = dr;
            w.hi = r;
            w.m_hi = m;
            ++r;
        }
    }
    return w;
}

__device__ __forceinline__ long long window_mult(const Window& w, int64_t e, int64_t j, long long cj) {
    return j == e ? w.m_self : (j == w.lo ? w.m_lo : (j == w.hi ? w.m_hi : cj));
}

// kPass 0: out = kdist.  kPass 1: prev = kdist, out = lrd.  kPass 2: prev = lrd, out = lof (may be null),
// verdict = lof > 1.5.
template <int kPass>
__global__ void __launch_bounds__(kThreads) k_lof_pass(const double* __restrict__ u, const int64_t* __restrict__ cnt,
                                                       int64_t D, int k, const double* __restrict__ prev,
                                                       double* __restrict__ out, uint8_t* __restrict__ verdict) {
    __shared__ double su[kStage];
    __shared__ long long sc[kStage];
    __shared__ double sx[kPass == 0 ? 1 : kStage];
    for (int64_t t0 = (int64_t)blockIdx.x * kTile; t0 < D; t0 += (int64_t)gridDim.x * kTile) {
        const int64_t base = t0 - k;
        const int64_t end = t0 + kTile + k < D ? t0 + kTile + k : D;
        const int n = (int)(end - base);
        __syncthreads();   // the previous tile has been consumed
        for (int t = threadIdx.x; t < n; t += kThreads) {
            const int64_t g = base + t;
            if (g < 0) continue;
            su[t] = __ldg(u + g);
            sc[t] = (long long)__ldg(cnt + g);
            if (kPass != 0) sx[t] = __ldg(prev + g);
        }
        __syncthreads();
#pragma unroll 1
        for (int q = 0; q < kPerThread; ++q) {
            const int64_t e = t0 + q * kThreads + threadIdx.x;
            if (e >= D) break;
            const Window w = lof_window(su, sc, base, e, D, k);
            if (kPass == 0) {
                out[e] = w.kdist;
                continue;
            }
            const double ue = su[e - base];
            double s = 0.0;
            for (int64_t j = w.lo; j <= w.hi; ++j) {
                const double m = (double)window_mult(w, e, j, sc[j - base]);
                double term;
                if (kPass == 1) {
                    const double d = j < e ? __dsub_rn(ue, su[j - base]) : (j > e ? __dsub_rn(su[j - base], ue) : 0.0);
                    const double kd = sx[j - base];
                    term = __dmul_rn(m, d > kd ? d : kd);
                } else {
                    term = __dmul_rn(m, __ddiv_rn(sx[j - base], sx[e - base]));
                }
                s = __dadd_rn(s, term);
            }
            const double mean = __ddiv_rn(s, (double)k);
            if (kPass == 1) {
                out[e] = __ddiv_rn(1.0, __dadd_rn(mean, 1e-10));
            } else {
                if (out) out[e] = mean;
                verdict[e] = mean > 1.5 ? 1 : 0;
            }
        }
    }
}

// Entry holding rank r of the expanded multiset: cum[i-1] <= r < cum[i] (inclusive prefix sums).
__global__ void __launch_bounds__(kThreads) k_find_ranks(const int64_t* __restrict__ cum, int64_t D, int64_t r0,
                                                         int64_t r1, int64_t* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < D; i += stride) {
        const int64_t lo = i ? cum[i - 1] : 0, hi = cum[i];
        if (lo <= r0 && r0 < hi) out[0] = i;
        if (lo <= r1 && r1 < hi) out[1] = i;
    }
}

}  // namespace

extern "C" {

int dr_lof_score(dr_ctx* ctx, const double* u, const int64_t* cnt, int64_t n_entries, int32_t k, uint8_t* verdict,
                 double* kdist, double* lrd, double* lof, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, k >= 1 && k <= kMaxK, "k must be in [1, 64]");
    if (n_entries <= 0) return DR_OK;
    DR_REQUIRE(ctx, u && cnt && verdict && kdist && lrd, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = dr_grid_for(ctx, n_entries, kTile, 4);
    k_lof_pass<0><<<grid, kThreads, 0, st>>>(u, cnt, n_entries, k, nullptr, kdist, nullptr);
    DR_LAUNCHED(ctx);
    k_lof_pass<1><<<grid, kThreads, 0, st>>>(u, cnt, n_entries, k, kdist, lrd, nullptr);
    DR_LAUNCHED(ctx);
    k_lof_pass<2><<<grid, kThreads, 0, st>>>(u, cnt, n_entries, k, lrd, lof, verdict);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_lof_median(dr_ctx* ctx, const int64_t* cnt, int64_t n_entries, int64_t r0, int64_t r1, int64_t* out_entry,
                  void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, out_entry, "null pointer");
    out_entry[0] = out_entry[1] = -1;
    if (n_entries <= 0) return DR_OK;
    DR_REQUIRE(ctx, cnt && r0 >= 0 && r1 >= 0, "null pointer / negative rank");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = dr_ensure_scratch(ctx, 2 * sizeof(int64_t));
    if (rc) return rc;
    int64_t* d_out = (int64_t*)ctx->scratch;
    int64_t* h_out = (int64_t*)ctx->pinned;
    int64_t* cum = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    DR_CUDA(ctx, cub::DeviceScan::InclusiveSum(nullptr, temp_bytes, cnt, cum, n_entries, st));
    DR_CUDA(ctx, cudaMallocAsync((void**)&cum, (size_t)n_entries * sizeof(int64_t) + temp_bytes, st));
    temp = cum + n_entries;
    cudaError_t e = cudaMemsetAsync(d_out, 0xff, 2 * sizeof(int64_t), st);
    if (e == cudaSuccess) e = cub::DeviceScan::InclusiveSum(temp, temp_bytes, cnt, cum, n_entries, st);
    ctx->launches++;
    if (e == cudaSuccess) {
        k_find_ranks<<<dr_grid_for(ctx, n_entries, kThreads, 8), kThreads, 0, st>>>(cum, n_entries, r0, r1, d_out);
        ctx->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_out, d_out, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(cum, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return dr_fail(ctx, DR_ERR_CUDA, "rank search failed: %s", cudaGetErrorString(e));
    out_entry[0] = h_out[0];
    out_entry[1] = h_out[1];
    return DR_OK;
}

}  // extern "C"
