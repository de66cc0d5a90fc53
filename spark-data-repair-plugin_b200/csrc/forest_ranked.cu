// dr_forest_predict_ranked: rank-coded forest inference for all-discrete models (see the header).
//
// Compared with the generic float64 kernel: a node is one 32-bit word instead of 12 bytes and a
// cell's features are two bytes each instead of eight, so a CTA of 256 cells needs ~17 KB of features
// and 16 warps stay resident per SM.  The forest is streamed through shared memory in chunks of whole
// trees by the TMA engine (cp.async.bulk, double buffered).  A warp waits on the buffer's mbarrier for
// the chunk to land and counts itself out when it is done with it; the last warp out starts the copy
// of the chunk two positions ahead -- no CTA-wide barrier in the loop and no producer thread polling
// (a version with a dedicated producer warp spent a large share of the issue slots in its wait loop; a ring of
// four half-size chunks was slower: the per-chunk bookkeeping doubles).  Each thread walks kIlp trees at a time for a fixed number of levels.  The kernel is bound
// by shared-memory wavefronts (two loads per level: rank byte, node word), so everything else is
// squeezed out of the level: the node word is carry coded (word + rank overflows into the child index
// exactly when the row goes right; siblings are adjacent), child indices are absolute within the
// chunk, leaves point at themselves and NaN is folded into the rank slots (one slot per (feature, NaN
// direction) that some node tests) -- a level is LDS, IADD, PRMT, LDS with no compare, select or
// branch.  The LAST level stops at the index of the node the walk ends on: leaf values are stored per
// node of each tree's tail (the host orders a tree's nodes so that all leaves sit there), so the leaf's
// own word is never loaded.  Leaf values are float64 and are added to the sequence's accumulator in
// tree order: margins are bit-identical to the generic kernel and to the oracle.
#include "common.cuh"

namespace {

// The kernel is bound by the shared-memory pipe, so what counts is wavefronts per level.  Two feature-tile layouts:
//  * wide   (1 CTA / SM): one 32-bit word per rank, [slot][thread].  Lane L of a warp always reads
//           bank L, whatever slot its node tests: the rank load is ONE wavefront (the byte layout
//           measures 1.96 once the lanes of a warp have spread over different nodes).
//           512 cells / CTA when n_slots * 2 KB fits beside the chunk buffers (<= 72 slots),
//           else 256 cells / CTA (<= 148 slots), then with more trees in flight per thread.
//  * bytes  (256 cells / CTA, 2 CTAs / SM when it fits): [thread][slot], odd word stride.
constexpr int kByteThreads = 256;
constexpr int kChunkNodes = DR_RANKED_CHUNK_NODES;
constexpr int kChunkLeaves = DR_RANKED_CHUNK_LEAVES;

struct RankedParams {
    dr_forest_ranked f;
    int32_t* tile;
    int n_cols;
    const int32_t* cells;
    int64_t n_cells;
    int target_col;
    double* out_margin;
    int feat_stride;  // bytes per thread row of the feature tile (multiple of 4, odd number of words)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// 1-D TMA bulk copy global -> shared, completion signalled on the mbarrier (16-byte granules)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// One level: two shared-memory loads (rank byte, next node word), one add and one byte extract.
// Addresses are 32-bit shared-window offsets (no generic-address arithmetic): in the wide layout
// feat = own column of the [slot][thread] word tile, so slot s sits at feat + s * 4 * T.
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
template <bool kWide, int T>
__device__ __forceinline__ uint32_t step_node(uint32_t nodes, uint32_t w, uint32_t feat, uint32_t lane_off) {
    uint32_t r;
    if (kWide) {
        // slot * (4 * T) + own column, as ONE multiply-add (left to itself the compiler turns the
        // shift pair into shift + mask and needs a third instruction for the add)
        uint32_t addr;
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(addr) : "r"(w >> 24), "n"(T * 4), "r"(feat + lane_off));
        r = lds_u32(addr);
    } else {
        r = lds_u8((w >> 24) + feat);
    }
    const uint32_t w2 = w + r;                                   // carries into bit 8 iff rank >= threshold
    return lds_u32(__byte_perm(w2, 0, 0x4421) * 4u + nodes);     // bits 8..23: left child (+1 = right child)
}

// Last level: only the index of the node the walk ends on (chunk relative).
template <bool kWide, int T>
__device__ __forceinline__ uint32_t last_node(uint32_t w, uint32_t feat, uint32_t lane_off) {
    uint32_t r;
    if (kWide) {
        uint32_t addr;
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(addr) : "r"(w >> 24), "n"(T * 4), "r"(feat + lane_off));
        r = lds_u32(addr);
    } else {
        r = lds_u8((w >> 24) + feat);
    }
    return __byte_perm(w + r, 0, 0x4421);
}

constexpr int kChunkTrees = DR_RANKED_CHUNK_TREES;

// value of chunk-relative leaf slot `at`: low and high word planes, kChunkLeaves words apart
__device__ __forceinline__ double leaf_value(uint32_t planes, int at) {
    const uint32_t a = planes + 4u * (uint32_t)at;
    uint32_t lo, hi;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(lo) : "r"(a));
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(hi) : "r"(a), "n"(DR_RANKED_CHUNK_LEAVES * 4));
    return __hiloint2double((int)hi, (int)lo);
}

struct __align__(16) ChunkBuf {
    // float64 leaf values as two planes of 32-bit words: a 64-bit load of 32 random leaves costs 3 wavefronts
    // (measured: leaves l and l + 16 of a tree share a bank pair), two 32-bit loads of <= 31 consecutive
    // words are conflict free, 2 wavefronts
    uint32_t leaf_lo[kChunkLeaves];
    uint32_t leaf_hi[kChunkLeaves];
    uint32_t node[kChunkNodes];
    uint2 hdr[kChunkTrees];  // per tree of the chunk: (root node word, value bias), chunk relative
};

constexpr int kStages = 2;  // chunk buffers in flight per CTA

template <bool kWide, int T, int kIlp>
__global__ void __launch_bounds__(T, kWide ? 1 : 2)
k_forest_predict_ranked(const __grid_constant__ RankedParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const dr_forest_ranked& F = p.f;
    ChunkBuf* buf = reinterpret_cast<ChunkBuf*>(smem_raw);                                // kStages chunk buffers
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + kStages * sizeof(ChunkBuf));  // chunk landed (per buffer)
    uint32_t* done = reinterpret_cast<uint32_t*>(full + kStages);                         // warps that left the buffer
    unsigned char* s_feat = smem_raw + kStages * sizeof(ChunkBuf) + kStages * 16;
    const int t = threadIdx.x;
    const int depth = F.max_depth;
    // Balanced partition: every CTA owns a contiguous, equal share of the cells and walks it in n_tiles
    // EQUAL tiles of tile_cells <= T cells (a multiple of 32).  A tile pass costs what its warps cost (the
    // kernel is bound by shared-memory wavefronts, i.e. by active warps), so a share of 845 cells is two
    // passes of 14 warps instead of a full one and a 333-cell one that both wait for every chunk: the
    // surplus warps of the CTA retire right after the set-up.  The CTA's chunk stream: every tile walks
    // chunks 0 .. n_chunks - 1; chunk k of the stream lives in buffer k % kStages.
    const int64_t c0 = (p.n_cells * (int64_t)blockIdx.x / (int64_t)gridDim.x + 31) & ~(int64_t)31;
    const int64_t c1_raw = (p.n_cells * ((int64_t)blockIdx.x + 1) / (int64_t)gridDim.x + 31) & ~(int64_t)31;
    const int64_t c1 = blockIdx.x + 1 == gridDim.x ? p.n_cells : (c1_raw < p.n_cells ? c1_raw : p.n_cells);
    const int64_t share = c1 > c0 ? c1 - c0 : 0;
    const uint32_t n_tiles = (uint32_t)((share + T - 1) / T);
    const int tile_cells = n_tiles ? (int)((((share + n_tiles - 1) / n_tiles) + 31) & ~(int64_t)31) : 0;
    const uint32_t n_warps = (uint32_t)(tile_cells / 32);   // warps that take part in the chunk hand-over
    const uint32_t n_stream = n_tiles * (uint32_t)F.n_chunks;

    auto issue = [&](uint32_t k) {  // one thread: start the TMA copies of stream chunk k
        const int c = (int)(k % (uint32_t)F.n_chunks), b = (int)(k % kStages);
        const int n0 = F.chunk_node_off[c], n1 = F.chunk_node_off[c + 1];
        const int l0 = F.chunk_leaf_off[c], l1 = F.chunk_leaf_off[c + 1];
        const int h0 = F.chunk_hdr_off[c], h1 = F.chunk_hdr_off[c + 1];
        const uint32_t nb = (uint32_t)(n1 - n0) * 4u, lb = (uint32_t)(l1 - l0) * 8u, hb = (uint32_t)(h1 - h0) * 8u;
        // (chunk_leaf_off is a multiple of 4: each plane of (l1 - l0) words is a whole number of 16-byte granules)
        mbar_expect_tx(&full[b], nb + lb + hb);
        bulk_g2s(buf[b].node, F.node_word + n0, nb, &full[b]);
        // chunk c's values sit at leaf_value[2 * l0 ..): its low words, then its high words
        bulk_g2s(buf[b].leaf_lo, F.leaf_value + 2 * (size_t)l0, lb / 2, &full[b]);
        bulk_g2s(buf[b].leaf_hi, F.leaf_value + 2 * (size_t)l0 + (size_t)(l1 - l0), lb / 2, &full[b]);
        bulk_g2s(buf[b].hdr, F.tree_hdr + 2 * (size_t)h0, hb, &full[b]);
    };

    if (t == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            done[s] = 0;
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (uint32_t k = 0; k < (uint32_t)kStages && k < n_stream; ++k) issue(k);
    }
    __syncthreads();  // the only CTA-wide barrier: from here on warps meet through the mbarriers / counters
    if (t >= tile_cells) return;  // (whole warps: tile_cells is a multiple of 32)

    // ---- consumer warps: one cell per thread; the feature tile is private to the thread ----
    unsigned char* my_feat = kWide ? s_feat + 4 * t : s_feat + (size_t)t * p.feat_stride;
    // wide: feat = the tile's base (uniform), lane_off = this thread's column; bytes: feat = own row
    const uint32_t feat = kWide ? smem_u32(s_feat) : smem_u32(my_feat);
    const uint32_t lane_off = 4u * (uint32_t)t;
    uint32_t k = 0;
    for (uint32_t tile = 0; tile < n_tiles; ++tile) {
        const int64_t i = c0 + (int64_t)tile * tile_cells + t;
        const bool live = i < c1;
        const bool warp_live = (i - (t & 31)) < c1;   // (warp-uniform: does lane 0 of this warp have a cell)
        const int64_t row = live ? p.cells[i] : 0;
        {
            // rank tile of this thread's cell (eight slots at a time, loads first: the tile row and the
            // rank look-ups are dependent global loads)
            const int32_t* trow = p.tile + row * p.n_cols;
            constexpr int kFill = 8;
            for (int s0 = 0; s0 < F.n_slots; s0 += kFill) {
                int code[kFill], lo[kFill], hi[kFill];
                uint8_t nanv[kFill];
#pragma unroll
                for (int j = 0; j < kFill; ++j) {
                    const int sl = s0 + j < F.n_slots ? s0 + j : F.n_slots - 1;
                    lo[j] = F.rank_lut_off[sl];
                    hi[j] = F.rank_lut_off[sl + 1];
                    nanv[j] = F.slot_nan[sl];
                    code[j] = live ? trow[F.slot_col[sl]] : -1;
                }
                uint8_t r[kFill];
#pragma unroll
                for (int j = 0; j < kFill; ++j) {
                    const int kk = lo[j] + code[j] + 1;
                    // a code outside the slot's LUT (e.g. the pmf modes' "unknown category") is NaN
                    r[j] = (kk >= lo[j] && kk < hi[j]) ? __ldg(F.rank_lut + kk) : nanv[j];
                }
#pragma unroll
                for (int j = 0; j < kFill; ++j) {
                    const int sl = s0 + j;
                    if (sl < F.n_slots) {
                        if (kWide) reinterpret_cast<uint32_t*>(my_feat)[sl * T] = r[j];
                        else       my_feat[sl] = r[j];
                    }
                }
            }
        }
        double best = 0.0, margin0 = 0.0, acc = F.baseline[0];
        int best_s = 0, cur_s = 0;
        // The leaf values of a group are only added (in tree order: bit-identical float64 sums) while
        // the NEXT group -- possibly of the next chunk -- walks its first level, so that the serial DADD
        // chain hides behind shared-memory latency instead of idling the warp.  A slot with nothing to add
        // holds -0.0: x + (-0.0) == x bit for bit for every x (also -0.0 and NaN), so the adds need no
        // per-tree test (a test and two selects per tree were ~4 % of the group's instructions).
        double pend[kIlp];
#pragma unroll
        for (int j = 0; j < kIlp; ++j) pend[j] = -0.0;
        for (int c = 0; c < F.n_chunks; ++c, ++k) {
            const int b = (int)(k % kStages);
            const int s = F.chunk_seq[c];
            if (s != cur_s) {  // previous sequence is complete
#pragma unroll
                for (int j = 0; j < kIlp; ++j) {
                    acc += pend[j];
                    pend[j] = -0.0;
                }
                if (live && p.out_margin) p.out_margin[i * F.n_seq + cur_s] = acc;
                if (cur_s == 0) { best = acc; margin0 = acc; }
                else if (acc > best) { best = acc; best_s = cur_s; }
                cur_s = s;
                acc = F.baseline[s];
            }
            while (!mbar_try_wait(&full[b], (k / kStages) & 1)) {}
            const uint32_t nodes = smem_u32(buf[b].node);
            const uint32_t leaves = smem_u32(buf[b].leaf_lo);
            const uint4* __restrict__ hdr4 = reinterpret_cast<const uint4*>(buf[b].hdr);
            // a warp without a live cell (the tail of the share's last tile) only takes part in the hand-over
            const int n_trees = warp_live ? F.chunk_tree_off[c + 1] - F.chunk_tree_off[c] : 0;
            for (int q = 0; q < n_trees; q += kIlp) {
                uint32_t w[kIlp];
                int lb[kIlp];
#pragma unroll
                for (int j = 0; j < kIlp; j += 2) {  // two tree headers per 128-bit broadcast load
                    const uint4 h = hdr4[(q + j) >> 1];
                    w[j] = h.x; lb[j] = (int)h.y; w[j + 1] = h.z; lb[j + 1] = (int)h.w;
                }
                if (q + kIlp > n_trees) {  // last group of a sequence: surplus slots re-walk tree 0
#pragma unroll
                    for (int j = 1; j < kIlp; ++j)
                        if (q + j >= n_trees) { w[j] = w[0]; lb[j] = lb[0]; }
                }
                // levels 1 .. depth-1: rank load + node load; the serial float64 adds of the PREVIOUS group
                // are issued between the loads of this group's first level
                if (depth > 1) {
#pragma unroll
                    for (int j = 0; j < kIlp; ++j) {
                        w[j] = step_node<kWide, T>(nodes, w[j], feat, lane_off);
                        acc += pend[j];
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < kIlp; ++j) acc += pend[j];
                }
                for (int d = 2; d < depth; ++d) {
#pragma unroll
                    for (int j = 0; j < kIlp; ++j) w[j] = step_node<kWide, T>(nodes, w[j], feat, lane_off);
                }
                // last level: the index of the final node is enough, its value is stored per node
                if (depth > 0) {
#pragma unroll
                    for (int j = 0; j < kIlp; ++j)
                        pend[j] = leaf_value(leaves, lb[j] + (int)last_node<kWide, T>(w[j], feat, lane_off));
                } else {
#pragma unroll
                    for (int j = 0; j < kIlp; ++j) pend[j] = leaf_value(leaves, lb[j] + (int)__byte_perm(w[j], 0, 0x4421));
                }
                if (q + kIlp > n_trees) {  // the surplus slots' values (tree 0 again) are not added
#pragma unroll
                    for (int j = 1; j < kIlp; ++j)
                        if (q + j >= n_trees) pend[j] = -0.0;
                }
            }
            // this warp is done with buffer b; the last warp to leave refills it with stream chunk
            // k + kStages (no producer thread, nobody polls)
            __syncwarp();
            if ((t & 31) == 0) {
                __threadfence_block();
                if (atomicAdd(&done[b], 1u) == n_warps - 1u) {
                    done[b] = 0;
                    __threadfence_block();
                    if (k + kStages < n_stream) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        issue(k + kStages);
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kIlp; ++j) acc += pend[j];  // the last group of the last sequence
        if (live && p.out_margin) p.out_margin[i * F.n_seq + cur_s] = acc;
        if (cur_s == 0) { best = acc; margin0 = acc; }
        else if (acc > best) { best = acc; best_s = cur_s; }
        if (live) {
            const int cls = F.n_seq == 1 ? (margin0 > 0.0 ? 1 : 0) : best_s;
            p.tile[row * p.n_cols + p.target_col] = cls < F.n_classes ? F.class_code[cls] : -1;
        }
    }
}

}  // namespace

extern "C" int dr_forest_predict_ranked(dr_ctx* ctx, const dr_forest_ranked* forest, int32_t* tile, int n_cols,
                                        const int32_t* cells, int64_t n_cells, int target_col, double* out_margin,
                                        void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    if (n_cells <= 0) return DR_OK;
    DR_REQUIRE(ctx, forest && cells && tile, "null pointer");
    const dr_forest_ranked& f = *forest;
    DR_REQUIRE(ctx, f.n_seq >= 1 && f.n_slots >= 0 && f.n_slots <= 255, "the ranked kernel takes at most 255 rank slots");
    DR_REQUIRE(ctx, f.baseline && f.slot_col && f.rank_lut_off && f.rank_lut && f.slot_nan && f.class_code &&
                        f.chunk_tree_off && f.chunk_seq && f.chunk_node_off && f.chunk_leaf_off && f.chunk_hdr_off &&
                        f.tree_hdr && f.node_word && f.leaf_value, "null forest array");
    DR_REQUIRE(ctx, f.n_chunks >= 1, "the ranked forest needs at least one chunk (one tree per sequence)");
    DR_REQUIRE(ctx, ((uintptr_t)f.node_word & 15) == 0 && ((uintptr_t)f.leaf_value & 15) == 0 &&
                        ((uintptr_t)f.tree_hdr & 15) == 0, "node / leaf / header arrays must be 16-byte aligned");
    DR_REQUIRE(ctx, f.max_depth >= 0 && f.max_depth <= 63, "bad max_depth");
    DR_REQUIRE(ctx, target_col >= 0 && target_col < n_cols, "bad target column");
    DR_REQUIRE(ctx, f.n_seq == 1 ? f.n_classes >= 2 : f.n_classes == f.n_seq, "class count mismatch");
    RankedParams p;
    p.f = f;
    p.tile = tile;
    p.n_cols = n_cols;
    p.cells = cells;
    p.n_cells = n_cells;
    p.target_col = target_col;
    p.out_margin = out_margin;
    // a leaf's self-loop reads (and ignores) rank slot 0: the tile always holds at least one slot
    const size_t fixed = kStages * sizeof(ChunkBuf) + kStages * 16;
    constexpr size_t kMaxSmem = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90
    const int n_slots = f.n_slots > 0 ? f.n_slots : 1;
    DR_REQUIRE(ctx, f.layout >= 0 && f.layout <= 3, "bad layout");
    const size_t smem_512 = fixed + (size_t)n_slots * 512 * 4, smem_256 = fixed + (size_t)n_slots * 256 * 4;
    const bool wide_ok = smem_256 <= kMaxSmem;
    if (f.layout >= 2 && !wide_ok)
        return dr_fail(ctx, DR_ERR_UNSUPPORTED, "the wide rank tile does not fit a forest with %d slots", f.n_slots);
    auto launch = [&](auto kernel, int threads, size_t smem, int per_sm) -> int {
        DR_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        // one warp's worth of cells is the unit of work (balanced partition in the kernel): a few thousand
        // cells spread over all SMs instead of filling a handful of 512-cell CTAs that each stream the whole
        // forest alone -- so that the launch of an FD-flagged target (~10^4 cells) does not cost what a large one does
        const int grid = dr_grid_for(ctx, n_cells, 32, per_sm);
        kernel<<<grid, threads, smem, (cudaStream_t)stream>>>(p);
        return DR_OK;
    };
    if (wide_ok && f.layout != 1) {
        p.feat_stride = 0;
        int rc;
        if (smem_512 <= kMaxSmem && f.layout == 0) rc = launch(k_forest_predict_ranked<true, 512, 8>, 512, smem_512, 1);
        else if (f.layout == 2)     rc = launch(k_forest_predict_ranked<true, 256, 8>, 256, smem_256, 1);
        else                        rc = launch(k_forest_predict_ranked<true, 256, 16>, 256, smem_256, 1);
        if (rc != DR_OK) return rc;
    } else {
        int words = (n_slots + 3) / 4;
        if ((words & 1) == 0) ++words;  // odd word stride: consecutive threads land on different banks
        p.feat_stride = words * 4;
        const size_t smem = fixed + (size_t)kByteThreads * p.feat_stride;
        if (smem > kMaxSmem)
            return dr_fail(ctx, DR_ERR_UNSUPPORTED, "ranked forest with %d slots exceeds shared memory", f.n_slots);
        const int rc = launch(k_forest_predict_ranked<false, kByteThreads, 8>, kByteThreads, smem,
                              smem <= 110 * 1024 ? 2 : 1);
        if (rc != DR_OK) return rc;
    }
    DR_LAUNCHED(ctx);
    return DR_OK;
}
