// Detector scans other than the NULL scan: LUT (regex / domain values), IQR range, exact
// quartiles, denial constraints, discretisation.  All are single streaming passes over 1..m
// columns (HBM-bound, 4 or 8 bytes per row and column in, 1 bit per row out).
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kCtasPerSm = 8;

// Evaluate `pred(row)` for every row and OR the resulting bits into `bm`.  Each 32-row word is
// produced by exactly one warp (ballot); it is merged with a fire-and-forget RED.OR.
template <class Pred>
__device__ __forceinline__ void rows_to_bitmap(int64_t n_rows, uint32_t* __restrict__ bm, Pred pred) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_pad = (n_rows + 31) & ~(int64_t)31;
    constexpr int kUnroll = 4;   // four independent rows per thread: their loads are in flight together
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; r + (kUnroll - 1) * stride < n_pad; r += kUnroll * stride) {
        bool bit[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t rr = r + j * stride;
            bit[j] = rr < n_rows ? pred(rr) : false;
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const unsigned w = __ballot_sync(0xffffffffu, bit[j]);
            if (lane == 0 && w != 0) atomicOr(bm + ((r + j * stride) >> 5), w);  // RED.OR: no load stall
        }
    }
    for (; r < n_pad; r += stride) {
        const bool bit = r < n_rows ? pred(r) : false;
        const unsigned w = __ballot_sync(0xffffffffu, bit);
        if (lane == 0 && w != 0) atomicOr(bm + (r >> 5), w);
    }
}

// null_hit: whether a NULL cell (code < 0) is flagged -- always for the LUT detectors, the verdict of the
// median's entry for LOF (NULL cells are filled with the median)
__global__ void __launch_bounds__(kThreads) k_lut_scan(const int32_t* __restrict__ col, int64_t n_rows,
                                                       const uint8_t* __restrict__ lut, int dict_size, bool null_hit,
                                                       uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        const int c = __ldcs(col + r);
        return c < 0 ? null_hit : (c < dict_size && __ldg(lut + c) != 0);
    });
}

__global__ void __launch_bounds__(kThreads) k_range_flag(const double* __restrict__ col, int64_t n_rows,
                                                         double lower, double upper, uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        const double v = __ldcs(col + r);
        return v < lower || v > upper;  // NaN compares false: NULLs are never outliers
    });
}

struct ConstParams {
    const int32_t* cols[DR_MAX_COLS];
    int32_t ops[DR_MAX_COLS];
    int32_t args[DR_MAX_COLS];
    int n_preds;
};

__global__ void __launch_bounds__(kThreads) k_dc_const(const __grid_constant__ ConstParams p, int64_t n_rows,
                                                       uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        bool ok = true;
        for (int i = 0; i < p.n_preds && ok; ++i) {
            const int c = __ldcs(p.cols[i] + r);
            const int a = p.args[i];
            switch (p.ops[i]) {
                case DR_OP_EQ: ok = c == a; break;
                case DR_OP_IQ: ok = c != a; break;
                case DR_OP_LT: ok = c >= 0 && c < a; break;
                default: ok = c >= 0 && c >= a; break;
            }
        }
        return ok;
    });
}

struct KeyParams {
    const int32_t* cols[DR_MAX_COLS];
    int64_t strides[DR_MAX_COLS];
    int n_keys;
};

__device__ __forceinline__ int64_t row_key(const KeyParams& k, int64_t r) {
    int64_t key = 0;
    for (int i = 0; i < k.n_keys; ++i) key += (int64_t)(__ldcs(k.cols[i] + r) + 1) * k.strides[i];
    return key;
}

// min / max of (b + 1) per NULL-safe key.  The tables are read first through L2 (ld.cg) so that the
// common case -- the value is already inside [lo, hi] -- costs no atomic at all.
__global__ void __launch_bounds__(kThreads) k_dc_fd_build(const __grid_constant__ KeyParams k,
                                                          const int32_t* __restrict__ b_col, int64_t n_rows,
                                                          int64_t key_space, int32_t* lo, int32_t* hi) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
        const int64_t key = row_key(k, r);
        if (key < 0 || key >= key_space) continue;
        const int v = __ldcs(b_col + r) + 1;
        if (v < __ldcg(lo + key)) atomicMin(lo + key, v);
        if (v > __ldcg(hi + key)) atomicMax(hi + key, v);
    }
}

// Small key spaces (the usual case: an FD on a categorical attribute): every CTA keeps private
// lo / hi tables in shared memory, where the already-in-range test is a plain LDS and the rare update a
// shared-memory atomic; the tables are merged into the global ones once per CTA.  Without this, 10^8
// rows hammer a few dozen L2 addresses.
constexpr int kSmemKeySpace = 8192;

__global__ void __launch_bounds__(kThreads) k_dc_fd_build_smem(const __grid_constant__ KeyParams k,
                                                               const int32_t* __restrict__ b_col, int64_t n_rows,
                                                               int key_space, int32_t* lo, int32_t* hi) {
    extern __shared__ int32_t s_tab[];
    int32_t* s_lo = s_tab;
    int32_t* s_hi = s_tab + key_space;
    for (int i = threadIdx.x; i < key_space; i += kThreads) { s_lo[i] = INT32_MAX; s_hi[i] = INT32_MIN; }
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    constexpr int kUnroll = 4;   // loads of four rows first, then the table checks
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; r + (kUnroll - 1) * stride < n_rows; r += kUnroll * stride) {
        int64_t key[kUnroll];
        int v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            key[j] = row_key(k, r + j * stride);
            v[j] = __ldcs(b_col + r + j * stride) + 1;
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            if (key[j] < 0 || key[j] >= key_space) continue;
            if (v[j] < s_lo[key[j]]) atomicMin(s_lo + key[j], v[j]);
            if (v[j] > s_hi[key[j]]) atomicMax(s_hi + key[j], v[j]);
        }
    }
    for (; r < n_rows; r += stride) {
        const int64_t key = row_key(k, r);
        if (key < 0 || key >= key_space) continue;
        const int v = __ldcs(b_col + r) + 1;
        if (v < s_lo[key]) atomicMin(s_lo + key, v);
        if (v > s_hi[key]) atomicMax(s_hi + key, v);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < key_space; i += kThreads) {
        if (s_lo[i] != INT32_MAX) atomicMin(lo + i, s_lo[i]);
        if (s_hi[i] != INT32_MIN) atomicMax(hi + i, s_hi[i]);
    }
}

__global__ void __launch_bounds__(kThreads) k_dc_fd_flag(const __grid_constant__ KeyParams k, int64_t n_rows,
                                                         int64_t key_space, const int32_t* __restrict__ lo,
                                                         const int32_t* __restrict__ hi, uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        const int64_t key = row_key(k, r);
        if (key < 0 || key >= key_space) return false;
        return __ldg(lo + key) != __ldg(hi + key);
    });
}

// EQ(a..) & LT(t1.x, t2.x): a row is matched iff some row of its key group has a larger x, i.e. iff
// x + 1 < max(x + 1) of the group (NULL never compares true: it is neither flagged nor the maximum)
__global__ void __launch_bounds__(kThreads) k_dc_lt_flag(const __grid_constant__ KeyParams k,
                                                         const int32_t* __restrict__ x, int64_t n_rows,
                                                         int64_t key_space, const int32_t* __restrict__ hi,
                                                         uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        const int v = x[r];
        if (v < 0) return false;
        const int64_t key = row_key(k, r);
        if (key < 0 || key >= key_space) return false;
        return v + 1 < __ldg(hi + key);
    });
}

// ---- key spaces too large for direct tables: open-addressing hash table keyed by the 64-bit key ----
// slot = (key, lo, hi); the key is claimed with a 64-bit CAS, lo / hi are the same idempotent min / max.
__device__ __forceinline__ uint64_t mix64(uint64_t x) {  // splitmix64 finaliser
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

__global__ void __launch_bounds__(kThreads) k_dc_hash_build(const __grid_constant__ KeyParams k,
                                                            const int32_t* __restrict__ b_col, int64_t n_rows,
                                                            unsigned long long* __restrict__ keys,
                                                            int32_t* __restrict__ lo, int32_t* __restrict__ hi,
                                                            uint64_t mask) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
        const unsigned long long key = (unsigned long long)row_key(k, r);
        const int v = __ldcs(b_col + r) + 1;
        uint64_t h = mix64(key) & mask;
        while (true) {
            unsigned long long cur = keys[h];
            if (cur == ~0ull) cur = atomicCAS(keys + h, ~0ull, key);  // claim an empty slot
            if (cur == ~0ull || cur == key) {
                if (v < __ldcg(lo + h)) atomicMin(lo + h, v);
                if (v > __ldcg(hi + h)) atomicMax(hi + h, v);
                break;
            }
            h = (h + 1) & mask;
        }
    }
}

// mode 0: lo != hi (EQ.. & IQ(b));  mode 1: x + 1 < hi (EQ.. & LT(x))
__global__ void __launch_bounds__(kThreads) k_dc_hash_flag(const __grid_constant__ KeyParams k,
                                                           const int32_t* __restrict__ x, int mode, int64_t n_rows,
                                                           const unsigned long long* __restrict__ keys,
                                                           const int32_t* __restrict__ lo,
                                                           const int32_t* __restrict__ hi, uint64_t mask,
                                                           uint32_t* __restrict__ bm) {
    rows_to_bitmap(n_rows, bm, [&](int64_t r) {
        const int v = mode == 1 ? x[r] : 0;
        if (mode == 1 && v < 0) return false;
        const unsigned long long key = (unsigned long long)row_key(k, r);
        uint64_t h = mix64(key) & mask;
        while (true) {
            const unsigned long long cur = __ldg(keys + h);
            if (cur == key) return mode == 1 ? v + 1 < __ldg(hi + h) : __ldg(lo + h) != __ldg(hi + h);
            if (cur == ~0ull) return false;  // (cannot happen for a row that was inserted)
            h = (h + 1) & mask;
        }
    });
}

__global__ void __launch_bounds__(kThreads) k_discretize(const double* __restrict__ vals, int64_t n_rows,
                                                         double vmin, double denom, int thres,
                                                         int32_t* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
        const double v = __ldcs(vals + r);
        int o = -1;
        if (v == v && denom != 0.0) {
            // (v - min) / (max - min) * thres, evaluated in this order in IEEE double, then int()
            const double q = __dmul_rn(__ddiv_rn(__dsub_rn(v, vmin), denom), (double)thres);
            o = (int)trunc(q);
        }
        out[r] = o;
    }
}

// ---- exact quartiles: MSD radix select over order-preserving 64-bit keys ----------------------
__device__ __forceinline__ unsigned long long f64_key(double v) {
    unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

constexpr int kDigitBits = 11;
constexpr int kBuckets = 1 << kDigitBits;
constexpr int kMaxStates = 4;

struct SelectParams {
    unsigned long long prefix[kMaxStates];
    unsigned long long mask;  // bits already fixed
    int shift;                // position of the digit examined in this pass
    int digit_mask;
    int n_states;
};

__global__ void __launch_bounds__(kThreads) k_radix_hist(const double* __restrict__ col, int64_t n_rows,
                                                         const __grid_constant__ SelectParams p,
                                                         unsigned long long* __restrict__ out) {
    __shared__ unsigned int h[kMaxStates * kBuckets];
    for (int i = threadIdx.x; i < p.n_states * kBuckets; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += stride) {
        const double v = __ldcs(col + r);
        if (v != v) continue;
        const double vz = v == 0.0 ? 0.0 : v;  // -0.0 and 0.0 are one value
        const unsigned long long key = f64_key(vz);
        const int d = (int)((key >> p.shift) & (unsigned long long)p.digit_mask);
        for (int s = 0; s < p.n_states; ++s)
            if ((key & p.mask) == p.prefix[s]) atomicAdd(&h[s * kBuckets + d], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < p.n_states * kBuckets; i += blockDim.x)
        if (h[i]) atomicAdd(out + i, (unsigned long long)h[i]);
}

double key_to_f64(unsigned long long k) {
    unsigned long long u = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
    double d;
    memcpy(&d, &u, sizeof(d));
    return d;
}

}  // namespace

extern "C" {

int dr_lut_scan(dr_ctx* ctx, const int32_t* col, int64_t n_rows, const uint8_t* lut, int32_t dict_size,
                uint32_t* bitmap, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, col && bitmap && (lut || dict_size == 0), "null pointer");
    if (n_rows <= 0) return DR_OK;
    k_lut_scan<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        col, n_rows, lut, dict_size, true, bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_lof_flag(dr_ctx* ctx, const int32_t* col, int64_t n_rows, const uint8_t* verdict, int32_t dict_size,
                int32_t null_verdict, uint32_t* bitmap, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, col && bitmap && (verdict || dict_size == 0), "null pointer");
    if (n_rows <= 0) return DR_OK;
    k_lut_scan<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        col, n_rows, verdict, dict_size, null_verdict != 0, bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_range_flag(dr_ctx* ctx, const double* col, int64_t n_rows, double lower, double upper, uint32_t* bitmap,
                  void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, col && bitmap, "null pointer");
    if (n_rows <= 0) return DR_OK;
    k_range_flag<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        col, n_rows, lower, upper, bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_dc_const(dr_ctx* ctx, const int32_t* const* cols, const int32_t* ops, const int32_t* args, int n_preds,
                int64_t n_rows, uint32_t* row_bitmap, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, cols && ops && args && row_bitmap, "null pointer");
    DR_REQUIRE(ctx, n_preds >= 1 && n_preds <= DR_MAX_COLS, "n_preds must be in [1, 64]");
    if (n_rows <= 0) return DR_OK;
    ConstParams p;
    memset(&p, 0, sizeof(p));
    p.n_preds = n_preds;
    for (int i = 0; i < n_preds; ++i) {
        DR_REQUIRE(ctx, cols[i] != nullptr, "null column pointer");
        DR_REQUIRE(ctx, ops[i] >= DR_OP_EQ && ops[i] <= DR_OP_GT, "unknown predicate op");
        p.cols[i] = cols[i];
        p.ops[i] = ops[i];
        p.args[i] = args[i];
    }
    k_dc_const<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(p, n_rows,
                                                                                                      row_bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

static int fill_keys(dr_ctx* ctx, KeyParams* k, const int32_t* const* key_cols, const int64_t* strides,
                     int n_keys) {
    DR_REQUIRE(ctx, key_cols && strides, "null pointer");
    DR_REQUIRE(ctx, n_keys >= 1 && n_keys <= DR_MAX_COLS, "n_keys must be in [1, 64]");
    memset(k, 0, sizeof(*k));
    k->n_keys = n_keys;
    for (int i = 0; i < n_keys; ++i) {
        DR_REQUIRE(ctx, key_cols[i] != nullptr, "null key column");
        k->cols[i] = key_cols[i];
        k->strides[i] = strides[i];
    }
    return DR_OK;
}

int dr_dc_fd_build(dr_ctx* ctx, const int32_t* const* key_cols, const int64_t* strides, int n_keys,
                   const int32_t* b_col, int64_t n_rows, int64_t key_space, int32_t* lo, int32_t* hi,
                   void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, b_col && lo && hi && key_space > 0, "null pointer / empty key space");
    KeyParams k;
    int rc = fill_keys(ctx, &k, key_cols, strides, n_keys);
    if (rc) return rc;
    if (n_rows <= 0) return DR_OK;
    if (key_space <= kSmemKeySpace) {
        const size_t smem = (size_t)key_space * 2 * sizeof(int32_t);
        DR_CUDA(ctx, cudaFuncSetAttribute(k_dc_fd_build_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int per_sm = smem <= 24 * 1024 ? 8 : (smem <= 48 * 1024 ? 4 : 2);
        k_dc_fd_build_smem<<<dr_grid_for(ctx, n_rows, kThreads, per_sm), kThreads, smem, (cudaStream_t)stream>>>(
            k, b_col, n_rows, (int)key_space, lo, hi);
        DR_LAUNCHED(ctx);
        return DR_OK;
    }
    k_dc_fd_build<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        k, b_col, n_rows, key_space, lo, hi);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_dc_fd_flag(dr_ctx* ctx, const int32_t* const* key_cols, const int64_t* strides, int n_keys,
                  int64_t n_rows, int64_t key_space, const int32_t* lo, const int32_t* hi, uint32_t* row_bitmap,
                  void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, lo && hi && row_bitmap && key_space > 0, "null pointer / empty key space");
    KeyParams k;
    int rc = fill_keys(ctx, &k, key_cols, strides, n_keys);
    if (rc) return rc;
    if (n_rows <= 0) return DR_OK;
    k_dc_fd_flag<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        k, n_rows, key_space, lo, hi, row_bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_dc_hash_build(dr_ctx* ctx, const int32_t* const* key_cols, const int64_t* strides, int n_keys,
                     const int32_t* b_col, int64_t n_rows, int64_t capacity, uint64_t* table_keys, int32_t* lo,
                     int32_t* hi, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, b_col && table_keys && lo && hi, "null pointer");
    DR_REQUIRE(ctx, capacity >= 2 && (capacity & (capacity - 1)) == 0, "capacity must be a power of two");
    DR_REQUIRE(ctx, capacity >= 2 * n_rows, "capacity must be at least twice the number of rows");
    KeyParams k;
    int rc = fill_keys(ctx, &k, key_cols, strides, n_keys);
    if (rc) return rc;
    if (n_rows <= 0) return DR_OK;
    k_dc_hash_build<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        k, b_col, n_rows, (unsigned long long*)table_keys, lo, hi, (uint64_t)capacity - 1);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_dc_hash_flag(dr_ctx* ctx, const int32_t* const* key_cols, const int64_t* strides, int n_keys,
                    const int32_t* x_col, int mode, int64_t n_rows, int64_t capacity, const uint64_t* table_keys,
                    const int32_t* lo, const int32_t* hi, uint32_t* row_bitmap, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, table_keys && lo && hi && row_bitmap, "null pointer");
    DR_REQUIRE(ctx, mode == 0 || (mode == 1 && x_col), "mode 1 (LT) needs the compared column");
    DR_REQUIRE(ctx, capacity >= 2 && (capacity & (capacity - 1)) == 0, "capacity must be a power of two");
    KeyParams k;
    int rc = fill_keys(ctx, &k, key_cols, strides, n_keys);
    if (rc) return rc;
    if (n_rows <= 0) return DR_OK;
    k_dc_hash_flag<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        k, x_col, mode, n_rows, (const unsigned long long*)table_keys, lo, hi, (uint64_t)capacity - 1, row_bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_dc_lt_flag(dr_ctx* ctx, const int32_t* const* key_cols, const int64_t* strides, int n_keys,
                  const int32_t* x_col, int64_t n_rows, int64_t key_space, const int32_t* hi, uint32_t* row_bitmap,
                  void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, x_col && hi && row_bitmap, "null pointer");
    KeyParams k;
    int rc = fill_keys(ctx, &k, key_cols, strides, n_keys);
    if (rc) return rc;
    if (n_rows <= 0) return DR_OK;
    k_dc_lt_flag<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        k, x_col, n_rows, key_space, hi, row_bitmap);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_discretize(dr_ctx* ctx, const double* vals, int64_t n_rows, double vmin, double denom, int32_t thres,
                  int32_t* out, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, vals && out, "null pointer");
    if (n_rows <= 0) return DR_OK;
    k_discretize<<<dr_grid_for(ctx, n_rows, kThreads, kCtasPerSm), kThreads, 0, (cudaStream_t)stream>>>(
        vals, n_rows, vmin, denom, thres, out);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

// Exact Spark `percentile` at 0.25 / 0.75: needs the order statistics floor(p(n-1)) and ceil(p(n-1)).
// Six histogram passes (11+11+11+11+10+10 bits) narrow up to four prefixes at once.
int dr_quartiles(dr_ctx* ctx, const double* col, int64_t n_rows, double* out_q, int64_t* out_n, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, col && out_q && out_n, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    out_q[0] = out_q[1] = NAN;
    *out_n = 0;
    if (n_rows <= 0) return DR_OK;
    int rc = dr_ensure_scratch(ctx, sizeof(unsigned long long) * kMaxStates * kBuckets);
    if (rc) return rc;
    unsigned long long* d_hist = (unsigned long long*)ctx->scratch;
    static thread_local unsigned long long h_hist[kMaxStates * kBuckets];
    const int grid = dr_grid_for(ctx, n_rows, kThreads, 4);

    // state = (prefix, remaining rank); several target ranks may share a state
    unsigned long long prefix[kMaxStates] = {0, 0, 0, 0};
    int64_t rank[kMaxStates] = {0, 0, 0, 0};  // rank inside the state's prefix bucket
    int state_of[4] = {0, 0, 0, 0};
    int n_states = 1;
    int64_t n = -1;
    double pos[2];
    int64_t want[4];
    unsigned long long mask = 0;
    const int widths[6] = {11, 11, 11, 11, 10, 10};
    int shift = 64;
    for (int pass = 0; pass < 6; ++pass) {
        shift -= widths[pass];
        SelectParams p;
        memset(&p, 0, sizeof(p));
        p.mask = mask;
        p.shift = shift;
        p.digit_mask = (1 << widths[pass]) - 1;
        p.n_states = n_states;
        for (int s = 0; s < n_states; ++s) p.prefix[s] = prefix[s];
        DR_CUDA(ctx, cudaMemsetAsync(d_hist, 0, sizeof(unsigned long long) * n_states * kBuckets, st));
        k_radix_hist<<<grid, kThreads, 0, st>>>(col, n_rows, p, d_hist);
        DR_LAUNCHED(ctx);
        DR_CUDA(ctx, cudaMemcpyAsync(h_hist, d_hist, sizeof(unsigned long long) * n_states * kBuckets,
                                     cudaMemcpyDeviceToHost, st));
        DR_CUDA(ctx, cudaStreamSynchronize(st));
        if (pass == 0) {
            n = 0;
            for (int b = 0; b < kBuckets; ++b) n += (int64_t)h_hist[b];
            *out_n = n;
            if (n == 0) return DR_OK;
            pos[0] = (double)(n - 1) * 0.25;
            pos[1] = (double)(n - 1) * 0.75;
            want[0] = (int64_t)floor(pos[0]);
            want[1] = (int64_t)ceil(pos[0]);
            want[2] = (int64_t)floor(pos[1]);
            want[3] = (int64_t)ceil(pos[1]);
        }
        // advance every target rank into its digit bucket, then rebuild the distinct states
        unsigned long long new_prefix[4];
        int64_t new_rank[4];
        for (int t = 0; t < 4; ++t) {
            const int s = state_of[t];
            int64_t k = pass == 0 ? want[t] : rank[t];
            const unsigned long long* hh = h_hist + (size_t)s * kBuckets;
            int b = 0;
            for (; b < (1 << widths[pass]); ++b) {
                if (k < (int64_t)hh[b]) break;
                k -= (int64_t)hh[b];
            }
            if (b == (1 << widths[pass])) return dr_fail(ctx, DR_ERR_CUDA, "radix select lost its rank");
            new_prefix[t] = prefix[s] | ((unsigned long long)b << shift);
            new_rank[t] = k;
        }
        mask |= ((unsigned long long)p.digit_mask) << shift;
        // rebuild the distinct states (several ranks may share a prefix)
        unsigned long long uniq[4];
        int nu = 0;
        for (int t = 0; t < 4; ++t) {
            int s = 0;
            for (; s < nu; ++s)
                if (uniq[s] == new_prefix[t]) break;
            if (s == nu) uniq[nu++] = new_prefix[t];
            state_of[t] = s;
            rank[t] = new_rank[t];
        }
        for (int s = 0; s < nu; ++s) prefix[s] = uniq[s];
        n_states = nu;
    }
    double v[4];
    for (int t = 0; t < 4; ++t) v[t] = key_to_f64(prefix[state_of[t]]);
    for (int q = 0; q < 2; ++q) {
        const double lo = floor(pos[q]), hi = ceil(pos[q]);
        // (higher - position) * v[lower] + (position - lower) * v[higher]
        out_q[q] = lo == hi ? v[2 * q] : (hi - pos[q]) * v[2 * q] + (pos[q] - lo) * v[2 * q + 1];
    }
    return DR_OK;
}

}  // extern "C"
