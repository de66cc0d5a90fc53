// Spark-compatible HyperLogLog++ registers (p = 9, 512 registers; oracle/hll.py is the specification).
//   k_hll_dict:  one pass over a column's dictionary (every distinct non-NULL value once): XxHash64 with
//                seed 42 of each entry -> register max in shared memory -> one global atomicMax per
//                (CTA, register).  Registers are idempotent under max, so the dictionary is all it needs.
//   k_hll_pairs: struct(x, y) registers over a pair's presence bits: for every set bit (i, j) the hash is
//                XxHash64(y_j, seed = hx[i]) (a NULL slot passes its seed through).
// Strings are read from an Arrow-layout buffer (int64 offsets + bytes) with aligned 8-byte loads.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRegs = 512;
constexpr int kPairsPerLaunch = 32;
constexpr uint64_t P1 = 11400714785074694791ull, P2 = 14029467366897019727ull, P3 = 1609587929392839161ull,
                   P4 = 9650029242287828579ull, P5 = 2870177450012600261ull;

__device__ __forceinline__ uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t lane) { return rotl(acc + lane * P2, 31) * P1; }
__device__ __forceinline__ uint64_t fmix(uint64_t h) {
    h ^= h >> 33;
    h *= P2;
    h ^= h >> 29;
    h *= P3;
    return h ^ (h >> 32);
}

// `nbytes` (1..8) little-endian bytes at byte position `pos` of an 8-byte aligned buffer; only the aligned
// words that hold one of those bytes are read.
__device__ __forceinline__ uint64_t load_le(const uint8_t* __restrict__ base, int64_t pos, int nbytes) {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(base + (pos & ~(int64_t)7));
    const int sh = (int)(pos & 7) * 8;
    uint64_t v = __ldg(w) >> sh;
    if (sh + nbytes * 8 > 64) v |= __ldg(w + 1) << (64 - sh);
    return nbytes == 8 ? v : v & ((1ull << (nbytes * 8)) - 1);
}

__device__ uint64_t xxh64_bytes(const uint8_t* __restrict__ base, int64_t pos, int64_t len, uint64_t seed) {
    const int64_t end = pos + len;
    uint64_t h;
    if (len >= 32) {
        uint64_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
        for (; pos + 32 <= end; pos += 32) {
            v1 = xx_round(v1, load_le(base, pos, 8));
            v2 = xx_round(v2, load_le(base, pos + 8, 8));
            v3 = xx_round(v3, load_le(base, pos + 16, 8));
            v4 = xx_round(v4, load_le(base, pos + 24, 8));
        }
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h = (h ^ xx_round(0, v1)) * P1 + P4;
        h = (h ^ xx_round(0, v2)) * P1 + P4;
        h = (h ^ xx_round(0, v3)) * P1 + P4;
        h = (h ^ xx_round(0, v4)) * P1 + P4;
    } else {
        h = seed + P5;
    }
    h += (uint64_t)len;
    for (; pos + 8 <= end; pos += 8) {
        h ^= xx_round(0, load_le(base, pos, 8));
        h = rotl(h, 27) * P1 + P4;
    }
    if (pos + 4 <= end) {
        h ^= load_le(base, pos, 4) * P1;
        h = rotl(h, 23) * P2 + P3;
        pos += 4;
    }
    if (pos < end) {
        uint64_t tail = load_le(base, pos, (int)(end - pos));
        for (; pos < end; ++pos, tail >>= 8) {
            h ^= (tail & 0xff) * P5;
            h = rotl(h, 11) * P1;
        }
    }
    return fmix(h);
}

// hashInt / hashLong of Spark's XXH64 (= XXH64 of 4 / 8 little-endian bytes)
__device__ __forceinline__ uint64_t xxh64_u32(uint32_t v, uint64_t seed) {
    uint64_t h = seed + P5 + 4;
    h ^= (uint64_t)v * P1;
    return fmix(rotl(h, 23) * P2 + P3);
}
__device__ __forceinline__ uint64_t xxh64_u64(uint64_t v, uint64_t seed) {
    uint64_t h = seed + P5 + 8;
    h ^= xx_round(0, v);
    return fmix(rotl(h, 27) * P1 + P4);
}

// XxHash64Function.hash(entry i, type, seed); floats are normalised (-0.0 -> 0.0, NaN -> canonical NaN)
__device__ __forceinline__ uint64_t hash_entry(int kind, const void* __restrict__ data,
                                               const int64_t* __restrict__ off, int64_t i, uint64_t seed) {
    switch (kind) {
        case DR_HLL_STRING: {
            const int64_t a = __ldg(off + i), b = __ldg(off + i + 1);
            return xxh64_bytes(static_cast<const uint8_t*>(data), a, b - a, seed);
        }
        case DR_HLL_INT:
            return xxh64_u32((uint32_t)__ldg(static_cast<const int32_t*>(data) + i), seed);
        case DR_HLL_LONG:
            return xxh64_u64((uint64_t)__ldg(static_cast<const long long*>(data) + i), seed);
        case DR_HLL_FLOAT: {
            const float f = __ldg(static_cast<const float*>(data) + i);
            return xxh64_u32(f != f ? 0x7fc00000u : f == 0.0f ? 0u : __float_as_uint(f), seed);
        }
        default: {
            const double d = __ldg(static_cast<const double*>(data) + i);
            return xxh64_u64(d != d ? 0x7ff8000000000000ull : d == 0.0 ? 0ull : (uint64_t)__double_as_longlong(d),
                             seed);
        }
    }
}

__device__ __forceinline__ void reg_update(int* s_reg, uint64_t x) {
    const int idx = (int)(x >> 55);
    const int val = __clzll((long long)((x << 9) | (1ull << 8))) + 1;
    if (s_reg[idx] < val) atomicMax(&s_reg[idx], val);
}

__device__ __forceinline__ void flush(const int* s_reg, int32_t* regs) {
    __syncthreads();
    for (int r = threadIdx.x; r < kRegs; r += blockDim.x)
        if (s_reg[r]) atomicMax(&regs[r], s_reg[r]);
}

__global__ void __launch_bounds__(kThreads) k_hll_dict(int kind, const void* __restrict__ data,
                                                       const int64_t* __restrict__ off, int64_t n,
                                                       uint64_t* __restrict__ hashes, int32_t* __restrict__ regs) {
    __shared__ int s_reg[kRegs];
    for (int r = threadIdx.x; r < kRegs; r += blockDim.x) s_reg[r] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t x = hash_entry(kind, data, off, i, 42);
        if (hashes) hashes[i] = x;
        reg_update(s_reg, x);
    }
    flush(s_reg, regs);
}

struct PairBatch {
    dr_hll_pair pair[kPairsPerLaunch];
    int n_pairs;
};

// blockIdx.y: the pair; blockIdx.x strides over the pair's presence words.
__global__ void __launch_bounds__(kThreads) k_hll_pairs(const __grid_constant__ PairBatch b) {
    __shared__ int s_reg[kRegs];
    const dr_hll_pair& p = b.pair[blockIdx.y];
    for (int r = threadIdx.x; r < kRegs; r += blockDim.x) s_reg[r] = 0;
    __syncthreads();
    const int64_t ny = (int64_t)p.dom_y + 1, n_bits = ((int64_t)p.dom_x + 1) * ny, n_words = (n_bits + 31) / 32;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        uint32_t word = __ldg(p.bits + w);
        while (word) {
            const int64_t bit = w * 32 + __ffs(word) - 1;
            word &= word - 1;
            if (bit >= n_bits) break;
            const int64_t i = bit / ny, j = bit - i * ny;
            const uint64_t seed = i == 0 ? 42ull : __ldg(reinterpret_cast<const unsigned long long*>(p.hx) + i - 1);
            reg_update(s_reg, j == 0 ? seed : hash_entry(p.y_kind, p.y_data, p.y_off, j - 1, seed));
        }
    }
    flush(s_reg, p.regs);
}

}  // namespace

extern "C" {

int dr_hll_dict(dr_ctx* ctx, int32_t kind, const void* data, const int64_t* offsets, int64_t n, uint64_t* hashes,
                int32_t* regs, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, kind >= DR_HLL_STRING && kind <= DR_HLL_DOUBLE, "unknown value kind");
    DR_REQUIRE(ctx, regs, "null pointer");
    if (n <= 0) return DR_OK;
    DR_REQUIRE(ctx, data && (kind != DR_HLL_STRING || offsets), "null pointer");
    DR_REQUIRE(ctx, kind != DR_HLL_STRING || ((uintptr_t)data & 7) == 0, "string bytes must be 8-byte aligned");
    k_hll_dict<<<dr_grid_for(ctx, n, kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(kind, data, offsets, n, hashes,
                                                                                       regs);
    DR_LAUNCHED(ctx);
    return DR_OK;
}

int dr_hll_pairs(dr_ctx* ctx, const dr_hll_pair* pairs, int n_pairs, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, n_pairs >= 0 && (pairs || n_pairs == 0), "null pointer");
    int64_t max_words = 0;
    for (int q = 0; q < n_pairs; ++q) {
        const dr_hll_pair& p = pairs[q];
        DR_REQUIRE(ctx, p.dom_x >= 0 && p.dom_y >= 0 && p.bits && p.regs, "bad pair");
        DR_REQUIRE(ctx, p.y_kind >= DR_HLL_STRING && p.y_kind <= DR_HLL_DOUBLE, "unknown value kind");
        DR_REQUIRE(ctx, (p.dom_x == 0 || p.hx) && (p.dom_y == 0 || p.y_data), "null pointer");
        DR_REQUIRE(ctx, p.y_kind != DR_HLL_STRING || p.dom_y == 0 || (p.y_off && ((uintptr_t)p.y_data & 7) == 0),
                   "string bytes must be 8-byte aligned, with offsets");
        const int64_t w = (((int64_t)p.dom_x + 1) * ((int64_t)p.dom_y + 1) + 31) / 32;
        if (w > max_words) max_words = w;
    }
    const int gx = (int)std::min<int64_t>((max_words + kThreads - 1) / kThreads, 64);
    for (int q0 = 0; q0 < n_pairs; q0 += kPairsPerLaunch) {
        PairBatch b;
        b.n_pairs = std::min(kPairsPerLaunch, n_pairs - q0);
        for (int q = 0; q < b.n_pairs; ++q) b.pair[q] = pairs[q0 + q];
        k_hll_pairs<<<dim3(gx, b.n_pairs), kThreads, 0, (cudaStream_t)stream>>>(b);
        DR_LAUNCHED(ctx);
    }
    return DR_OK;
}

}  // extern "C"
