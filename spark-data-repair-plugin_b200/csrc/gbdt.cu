// dr_gbdt_train: histogram GBDT trainer on the GPU (SURVEY.md 8f "next" #1; replaces the LightGBM +
// hyperopt producer of train.py:89-229 with the reference's fixed parameters, see oracle/gbdt.py for
// the algorithm specification this file reproduces BIT FOR BIT).
//
// The training set of a repair model is tiny by GPU standards (<= max_training_row_num = 10 000 rows,
// <= ~100 pre-binned byte features), so the trainer is organised around launch count, not bandwidth:
// all S class-trees of a boosting round grow together, level by level, with a fixed launch sequence
// per round and NO host synchronisation until the whole forest is built:
//   k_grad      gradients / hessians of the objective, quantised to integers (exact histograms)
//   k_root      root sums
//   per level:  k_level (one CTA per (sequence, active leaf): shared-memory integer histogram of the
//               leaf's rows, then the leaf's best split), k_apply (one warp per sequence: picks the
//               proposals by decreasing gain under the num_leaves budget, creates children),
//               k_reassign (rows move to their child)
//   k_finish    leaf values, score update, tree nodes appended to the output
// dr_gbdt_train_ex adds the boosting options of oracle/gbdt_boost.py.  At their defaults it runs the
// loop above unchanged; otherwise a second loop of the same shape with
//   k_level<true> / k_finish_ex   reg_alpha (soft-thresholded G), min_split_gain, dart / rf leaf scaling
//   k_grad64, k_goss_select, k_goss_apply   goss: float64 gradients and row scores, exact top-k by a
//               single-CTA radix select, then the kept rows' amplified quantised gradients
//   k_bag       rf: gradients stay those of the initial scores, only the bag is redrawn
//   k_dart_walk, k_dart_scale   dart: dropped trees leave and re-enter the scores (walked over the
//               byte bins of the finished trees in out), their leaves rescaled in place
// The dart drop schedule is computed on the host beforehand, so this loop has no synchronisation either.
// Determinism: integer histograms are order independent; every floating-point expression uses
// explicit round-to-nearest intrinsics in the oracle's order (no FMA contraction); exp() is exp_det.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kMaxNodes = 64;   // num_leaves <= 32
constexpr int kMaxLeaves = 32;
constexpr int kThreads = 256;

struct Node {  // 16 bytes, output format (see dr_gbdt_node in the header)
    int16_t feature;  // -1 = leaf
    uint8_t thr_bin, missing_left, left, right;
    uint8_t pad[2];
    double value;
};

struct Proposal {
    double gain;
    int32_t feature, thr_bin, missing_left, leaf;
    long long GL, HL;
    int32_t CL;
};

struct GbdtState {
    // inputs
    const uint8_t* bins;   // [n][F]
    const int32_t* y_class;
    const double* y_value;
    const double* weight;
    int32_t n_bins[128];
    int32_t bin_off[129];
    int n, F, S, n_classes, max_depth, num_leaves, min_data;
    double lr, qscale, min_hess_q, factor, lam_q;
    int col_thr;           // colsample_bytree as a 24-bit threshold, -1 = every feature
    int bag_thr, bag_freq; // subsample as a 24-bit threshold, bagging period (0 = no bagging)
    unsigned long long seed;
    // workspace
    double* scores;        // [n][S]
    int32_t* gq;           // [S][n]
    int32_t* hq;           // [S][n]
    uint8_t* node_of;      // [S][n]
    uint8_t* inbag;        // [n] 1 = the row contributes to the trees of this iteration
    long long* sumG;       // [S][kMaxNodes]
    long long* sumH;
    int32_t* sumC;
    int32_t* active;       // [S][kMaxLeaves]
    int32_t* n_active;     // [S]
    int32_t* n_nodes;      // [S]
    int32_t* n_leaves;     // [S]
    Proposal* props;       // [S][kMaxLeaves]
    Node* cur;             // [S][kMaxNodes] tree under construction
    int32_t* split_flag;   // [S][kMaxNodes] 1 if the node was split at this level
    Node* out;             // [n_iter][S][kMaxNodes]
    int32_t* out_count;    // [n_iter][S]
    // boosting options (dr_gbdt_train_ex; all zero for plain gbdt)
    double alpha_q;        // reg_alpha * qscale
    double gain_floor;     // min_split_gain * qscale
    double rf_div;         // rf: leaf values are divided by n_iter (0 = scaled by the learning rate)
    int goss_top_k, goss_other_thr;  // goss: rows kept by score, 24-bit threshold of the other rows' draw
    double goss_amp;       // goss: (n - top_k) / other_k, the other rows' gradient factor
    double* g64;           // [S][n] goss: unquantised gradients
    double* h64;           // [S][n]
    double* rscore;        // [n] goss: sum over classes of |g * h|
    unsigned long long* goss_tau;  // goss: bits of the top_k-th largest row score
};

// splitmix64 finaliser (oracle/gbdt.py mix64): feature / row sub-sampling is a pure function of
// (seed, iteration, sequence, feature) resp. (seed, bag, row), identical on both sides
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ unsigned feat_hash(const unsigned long long seed, int it, int s, int f) {
    return (unsigned)(mix64(seed * 0x9E3779B97F4A7C15ull + ((unsigned long long)it << 40) +
                            ((unsigned long long)s << 20) + (unsigned long long)f + 1ull) >> 40);
}

__device__ __forceinline__ double exp_det(double x) {
    x = fmin(fmax(x, -700.0), 700.0);
    const double k = rint(__dmul_rn(x, 1.44269504088896338700e+00));
    const double r = __dsub_rn(__dsub_rn(x, __dmul_rn(k, 6.93147180369123816490e-01)),
                               __dmul_rn(k, 1.90821492927058770002e-10));
    const double c[14] = {1.0, 1.0, 1.0 / 2, 1.0 / 6, 1.0 / 24, 1.0 / 120, 1.0 / 720, 1.0 / 5040, 1.0 / 40320,
                          1.0 / 362880, 1.0 / 3628800, 1.0 / 39916800, 1.0 / 479001600, 1.0 / 6227020800.0};
    double p = c[13];
#pragma unroll
    for (int i = 12; i >= 0; --i) p = __dadd_rn(__dmul_rn(p, r), c[i]);
    return ldexp(p, (int)k);
}

// row i's bag membership, drawn every bag_freq iterations
__device__ __forceinline__ void draw_bag(const GbdtState& st, int iter, int i) {
    if (st.bag_freq > 0 && iter % st.bag_freq == 0) {  // a new bag every bag_freq iterations
        const unsigned long long bag = (unsigned long long)(iter / st.bag_freq);
        const unsigned h = (unsigned)(mix64((st.seed + 1ull) * 0x9E3779B97F4A7C15ull + (bag << 32) +
                                            (unsigned long long)i) >> 40);
        st.inbag[i] = h < (unsigned)st.bag_thr ? 1 : 0;
    }
}

// gradient and hessian of row i for every class k (ascending), handed to put(k, g, h)
template <class Put>
__device__ __forceinline__ void row_gradients(const GbdtState& st, int i, Put put) {
    const int S = st.S;
    const double* sc = st.scores + (size_t)i * S;
    if (st.n_classes == 1) {
        put(0, __dsub_rn(sc[0], st.y_value[i]), 1.0);
    } else if (st.n_classes == 2) {
        const double s = sc[0], w = st.weight[i], y = (double)st.y_class[i];
        const double e = exp_det(-fabs(s));
        const double p = s >= 0.0 ? __ddiv_rn(1.0, __dadd_rn(1.0, e)) : __ddiv_rn(e, __dadd_rn(1.0, e));
        put(0, __dmul_rn(__dsub_rn(p, y), w), __dmul_rn(__dmul_rn(p, __dsub_rn(1.0, p)), w));
    } else {
        double m = sc[0];
        for (int k = 1; k < S; ++k) m = fmax(m, sc[k]);
        double tot = 0.0;
        for (int k = 0; k < S; ++k) tot = __dadd_rn(tot, exp_det(__dsub_rn(sc[k], m)));
        const double w = st.weight[i];
        const int yc = st.y_class[i];
        for (int k = 0; k < S; ++k) {
            const double p = __ddiv_rn(exp_det(__dsub_rn(sc[k], m)), tot);
            put(k, __dmul_rn(__dsub_rn(p, k == yc ? 1.0 : 0.0), w),
                __dmul_rn(__dmul_rn(__dmul_rn(st.factor, p), __dsub_rn(1.0, p)), w));
        }
    }
}

__global__ void __launch_bounds__(kThreads) k_grad(GbdtState st, int iter) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st.n) return;
    draw_bag(st, iter, i);
    row_gradients(st, i, [&](int k, double g, double h) {
        st.gq[(size_t)k * st.n + i] = (int32_t)rint(__dmul_rn(g, st.qscale));
        st.hq[(size_t)k * st.n + i] = (int32_t)rint(__dmul_rn(h, st.qscale));
    });
    for (int k = 0; k < st.S; ++k) st.node_of[(size_t)k * st.n + i] = 0;
}

// rf after the first iteration: the gradients stay those of the initial scores, only the bag is redrawn
__global__ void __launch_bounds__(kThreads) k_bag(GbdtState st, int iter) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st.n) return;
    draw_bag(st, iter, i);
    for (int k = 0; k < st.S; ++k) st.node_of[(size_t)k * st.n + i] = 0;
}

// goss: unquantised gradients and the row score sum_k |g * h| (ascending class)
__global__ void __launch_bounds__(kThreads) k_grad64(GbdtState st) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st.n) return;
    double score = 0.0;
    row_gradients(st, i, [&](int k, double g, double h) {
        st.g64[(size_t)k * st.n + i] = g;
        st.h64[(size_t)k * st.n + i] = h;
        score = __dadd_rn(score, fabs(__dmul_rn(g, h)));
    });
    st.rscore[i] = score;
    for (int k = 0; k < st.S; ++k) st.node_of[(size_t)k * st.n + i] = 0;
}

// goss: the top_k-th largest row score, by a radix select over its IEEE bits (scores are >= 0, so the
// bits order like the values), one byte per pass from the most significant one
constexpr int kSelectThreads = 1024;
__global__ void __launch_bounds__(kSelectThreads) k_goss_select(GbdtState st) {
    __shared__ int hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_rank;
    const unsigned long long* bits = reinterpret_cast<const unsigned long long*>(st.rscore);
    if (threadIdx.x == 0) { s_prefix = 0; s_rank = st.goss_top_k; }
    unsigned long long mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += kSelectThreads) hist[b] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        for (int i = threadIdx.x; i < st.n; i += kSelectThreads) {
            const unsigned long long v = bits[i];
            if ((v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {  // the digit holding the rank-th largest of the rows matching the prefix
            int rank = s_rank, d = 255;
            for (; d > 0 && hist[d] < rank; --d) rank -= hist[d];
            s_rank = rank;
            s_prefix = prefix | ((unsigned long long)d << shift);
        }
        mask |= 255ull << shift;
        __syncthreads();
    }
    if (threadIdx.x == 0) *st.goss_tau = s_prefix;
}

// goss: rows scoring >= the top_k-th largest stay; every other row stays iff hash(seed, iter, i) falls
// below the threshold, its gradient and hessian amplified before quantisation
__global__ void __launch_bounds__(kThreads) k_goss_apply(GbdtState st, int iter) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st.n) return;
    const bool top = reinterpret_cast<const unsigned long long*>(st.rscore)[i] >= *st.goss_tau;
    const unsigned h = (unsigned)(mix64((st.seed + 2ull) * 0x9E3779B97F4A7C15ull + ((unsigned long long)iter << 32) +
                                        (unsigned long long)i) >> 40);
    st.inbag[i] = top || h < (unsigned)st.goss_other_thr ? 1 : 0;
    for (int k = 0; k < st.S; ++k) {
        double g = st.g64[(size_t)k * st.n + i], hs = st.h64[(size_t)k * st.n + i];
        if (!top) { g = __dmul_rn(g, st.goss_amp); hs = __dmul_rn(hs, st.goss_amp); }
        st.gq[(size_t)k * st.n + i] = (int32_t)rint(__dmul_rn(g, st.qscale));
        st.hq[(size_t)k * st.n + i] = (int32_t)rint(__dmul_rn(hs, st.qscale));
    }
}

// L1: T(G) = sign(G) * max(|G| - alpha_q, 0); at alpha_q = 0 exactly (double)G
__device__ __forceinline__ double soft_q(long long G, double alpha_q) {
    const double a = __dsub_rn(fabs((double)G), alpha_q);
    return a > 0.0 ? (G > 0 ? a : -a) : 0.0;
}

// one CTA per sequence: root sums + per-round tree state
__global__ void __launch_bounds__(kThreads) k_root(GbdtState st) {
    __shared__ long long sg[kThreads / 32], sh[kThreads / 32];
    __shared__ int sc[kThreads / 32];
    const int s = blockIdx.x;
    long long g = 0, h = 0;
    int c = 0;
    for (int i = threadIdx.x; i < st.n; i += kThreads) {
        if (!st.inbag[i]) continue;
        g += st.gq[(size_t)s * st.n + i];
        h += st.hq[(size_t)s * st.n + i];
        ++c;
    }
    for (int o = 16; o; o >>= 1) {
        g += __shfl_down_sync(0xffffffffu, g, o);
        h += __shfl_down_sync(0xffffffffu, h, o);
        c += __shfl_down_sync(0xffffffffu, c, o);
    }
    if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = g; sh[threadIdx.x >> 5] = h; sc[threadIdx.x >> 5] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long G = 0, H = 0;
        int C = 0;
        for (int j = 0; j < kThreads / 32; ++j) { G += sg[j]; H += sh[j]; C += sc[j]; }
        st.sumG[s * kMaxNodes] = G;
        st.sumH[s * kMaxNodes] = H;
        st.sumC[s * kMaxNodes] = C;
        st.active[s * kMaxLeaves] = 0;
        st.n_active[s] = 1;
        st.n_nodes[s] = 1;
        st.n_leaves[s] = 1;
        Node nd;
        nd.feature = -1; nd.thr_bin = 0; nd.missing_left = 0; nd.left = 0; nd.right = 0; nd.pad[0] = nd.pad[1] = 0;
        nd.value = 0.0;
        st.cur[s * kMaxNodes] = nd;
    }
}

// CTA (s, j): histogram of active leaf j of sequence s in shared memory, then its best split.
// kOpt: reg_alpha and min_split_gain (dr_gbdt_train_ex); k_level<false> is the plain trainer's
template <bool kOpt>
__global__ void __launch_bounds__(kThreads) k_level(GbdtState st, int iter) {
    extern __shared__ unsigned char smem_raw[];
    __shared__ unsigned s_fhash[128];
    __shared__ int s_fmin;
    const int s = blockIdx.x, j = blockIdx.y;
    Proposal* out = st.props + (s * kMaxLeaves + j);
    if (threadIdx.x == 0) { out->gain = 0.0; out->feature = -1; out->leaf = -1; }
    if (j >= st.n_active[s]) return;
    const int leaf = st.active[s * kMaxLeaves + j];
    const long long G = st.sumG[s * kMaxNodes + leaf], H = st.sumH[s * kMaxNodes + leaf];
    const int cnt = st.sumC[s * kMaxNodes + leaf];
    if (cnt < 2 * st.min_data || H <= 0) return;
    const int total = st.bin_off[st.F];
    // the host picks the quantisation so that every bin sum fits 32 bits: native shared-memory
    // atomics (64-bit ones degrade to compare-and-swap loops under the contention of few-valued features)
    int* hg = reinterpret_cast<int*>(smem_raw);
    int* hh = hg + total;
    int* hc = hh + total;
    for (int b = threadIdx.x; b < total; b += kThreads) { hg[b] = 0; hh[b] = 0; hc[b] = 0; }
    __syncthreads();
    const uint8_t* nof = st.node_of + (size_t)s * st.n;
    const int32_t* gq = st.gq + (size_t)s * st.n;
    const int32_t* hq = st.hq + (size_t)s * st.n;
    if (st.col_thr >= 0) {  // colsample_bytree: the features tree (iter, s) may split on
        if (threadIdx.x < st.F) s_fhash[threadIdx.x] = feat_hash(st.seed, iter, s, threadIdx.x);
        __syncthreads();
        if (threadIdx.x == 0) {
            int m = 0;
            for (int f = 1; f < st.F; ++f)
                if (s_fhash[f] < s_fhash[m]) m = f;
            s_fmin = m;
        }
    }
    for (int i = threadIdx.x; i < st.n; i += kThreads) {
        if (nof[i] != leaf || !st.inbag[i]) continue;
        const int g = gq[i], h = hq[i];
        const uint8_t* row = st.bins + (size_t)i * st.F;
        for (int f = 0; f < st.F; ++f) {
            const int b = st.bin_off[f] + row[f];
            atomicAdd(hg + b, g);
            atomicAdd(hh + b, h);
            atomicAdd(hc + b, 1);
        }
    }
    __syncthreads();
    // best split: thread f scans feature f in the oracle's order (t ascending, missing right then left)
    double best_gain = 0.0;
    int best_key = 0x7fffffff, best_f = -1, best_t = 0, best_ml = 0, best_CL = 0;
    long long best_GL = 0, best_HL = 0;
    double parent;
    if (kOpt) {
        const double t = soft_q(G, st.alpha_q);
        parent = __ddiv_rn(__dmul_rn(t, t), __dadd_rn((double)H, st.lam_q));
    } else {
        parent = __ddiv_rn(__dmul_rn((double)G, (double)G), __dadd_rn((double)H, st.lam_q));
    }
    for (int f = threadIdx.x; f < st.F; f += kThreads) {
        const int nb = st.n_bins[f];
        if (nb < 3) continue;
        if (st.col_thr >= 0 && !(s_fhash[f] < (unsigned)st.col_thr || f == s_fmin)) continue;
        const int o = st.bin_off[f];
        const long long mg = hg[o + nb - 1], mh = hh[o + nb - 1];
        const int mc = hc[o + nb - 1];
        long long cg = 0, ch = 0;
        int cc = 0;
        for (int t = 0; t < nb - 2; ++t) {
            cg += hg[o + t]; ch += hh[o + t]; cc += hc[o + t];
            for (int ml = 0; ml < 2; ++ml) {
                const long long GL = ml ? cg + mg : cg, HL = ml ? ch + mh : ch;
                const int CL = ml ? cc + mc : cc;
                const long long GR = G - GL, HR = H - HL;
                const int CR = cnt - CL;
                if (CL < st.min_data || CR < st.min_data) continue;
                if ((double)HL < st.min_hess_q || (double)HR < st.min_hess_q) continue;
                double gain;
                if (kOpt) {
                    const double tl = soft_q(GL, st.alpha_q), tr = soft_q(GR, st.alpha_q);
                    gain = __dsub_rn(__dadd_rn(__ddiv_rn(__dmul_rn(tl, tl), __dadd_rn((double)HL, st.lam_q)),
                                               __ddiv_rn(__dmul_rn(tr, tr), __dadd_rn((double)HR, st.lam_q))), parent);
                } else {
                    gain = __dsub_rn(
                        __dadd_rn(__ddiv_rn(__dmul_rn((double)GL, (double)GL), __dadd_rn((double)HL, st.lam_q)),
                                  __ddiv_rn(__dmul_rn((double)GR, (double)GR), __dadd_rn((double)HR, st.lam_q))),
                        parent);
                }
                if (gain > 0.0 && gain > best_gain) {
                    best_gain = gain; best_f = f; best_t = t; best_ml = ml;
                    best_key = (f << 16) | (t << 1) | ml;
                    best_GL = GL; best_HL = HL; best_CL = CL;
                }
            }
        }
    }
    // block arg-max: larger gain wins, ties go to the smaller (f, t, ml) key = the oracle's scan order
    __shared__ double r_gain[kThreads];
    __shared__ int r_key[kThreads];
    r_gain[threadIdx.x] = best_f >= 0 ? best_gain : -1.0;
    r_key[threadIdx.x] = best_key;
    __syncthreads();
    for (int o = kThreads / 2; o; o >>= 1) {
        if (threadIdx.x < o) {
            const double ga = r_gain[threadIdx.x], gb = r_gain[threadIdx.x + o];
            const int ka = r_key[threadIdx.x], kb = r_key[threadIdx.x + o];
            if (gb > ga || (gb == ga && kb < ka)) { r_gain[threadIdx.x] = gb; r_key[threadIdx.x] = kb; }
        }
        __syncthreads();
    }
    if (best_f >= 0 && r_gain[0] == best_gain && r_key[0] == best_key && (!kOpt || best_gain > st.gain_floor)) {
        out->gain = best_gain; out->feature = best_f; out->thr_bin = best_t; out->missing_left = best_ml;
        out->leaf = leaf; out->GL = best_GL; out->HL = best_HL; out->CL = best_CL;
    }
}

// one thread per sequence: apply proposals by decreasing gain (ties: smaller leaf id) under the budget
__global__ void k_apply(GbdtState st, int depth) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= st.S) return;
    const int na = st.n_active[s];
    for (int n = 0; n < kMaxNodes; ++n) st.split_flag[s * kMaxNodes + n] = 0;
    Proposal* pr = st.props + s * kMaxLeaves;
    bool used[kMaxLeaves];
    for (int j = 0; j < kMaxLeaves; ++j) used[j] = false;
    int new_active[kMaxLeaves];
    int n_new = 0;
    int n_nodes = st.n_nodes[s], n_leaves = st.n_leaves[s];
    for (int round = 0; round < na; ++round) {
        int pick = -1;
        for (int j = 0; j < na; ++j) {
            if (used[j] || pr[j].feature < 0 || !(pr[j].gain > 0.0)) continue;
            if (pick < 0 || pr[j].gain > pr[pick].gain || (pr[j].gain == pr[pick].gain && pr[j].leaf < pr[pick].leaf))
                pick = j;
        }
        if (pick < 0 || n_leaves >= st.num_leaves) break;
        used[pick] = true;
        const Proposal p = pr[pick];
        const int leaf = p.leaf, li = n_nodes, ri = n_nodes + 1;
        n_nodes += 2;
        n_leaves += 1;
        Node* cur = st.cur + s * kMaxNodes;
        cur[leaf].feature = (int16_t)p.feature; cur[leaf].thr_bin = (uint8_t)p.thr_bin;
        cur[leaf].missing_left = (uint8_t)p.missing_left; cur[leaf].left = (uint8_t)li; cur[leaf].right = (uint8_t)ri;
        Node nd;
        nd.feature = -1; nd.thr_bin = 0; nd.missing_left = 0; nd.left = 0; nd.right = 0; nd.pad[0] = nd.pad[1] = 0;
        nd.value = 0.0;
        cur[li] = nd; cur[ri] = nd;
        const long long G = st.sumG[s * kMaxNodes + leaf], H = st.sumH[s * kMaxNodes + leaf];
        const int cnt = st.sumC[s * kMaxNodes + leaf];
        st.sumG[s * kMaxNodes + li] = p.GL; st.sumH[s * kMaxNodes + li] = p.HL; st.sumC[s * kMaxNodes + li] = p.CL;
        st.sumG[s * kMaxNodes + ri] = G - p.GL; st.sumH[s * kMaxNodes + ri] = H - p.HL;
        st.sumC[s * kMaxNodes + ri] = cnt - p.CL;
        st.split_flag[s * kMaxNodes + leaf] = 1;
        new_active[n_new++] = li;
        new_active[n_new++] = ri;
    }
    st.n_nodes[s] = n_nodes;
    st.n_leaves[s] = n_leaves;
    const bool more = depth + 1 < st.max_depth;
    st.n_active[s] = more ? n_new : 0;
    for (int j = 0; j < n_new && j < kMaxLeaves; ++j) st.active[s * kMaxLeaves + j] = new_active[j];
}

__global__ void __launch_bounds__(kThreads) k_reassign(GbdtState st) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (i >= st.n) return;
    const int node = st.node_of[(size_t)s * st.n + i];
    if (!st.split_flag[s * kMaxNodes + node]) return;
    const Node nd = st.cur[s * kMaxNodes + node];
    const int b = st.bins[(size_t)i * st.F + nd.feature];
    const bool go_left = b == st.n_bins[nd.feature] - 1 ? nd.missing_left == 1 : b <= nd.thr_bin;
    st.node_of[(size_t)s * st.n + i] = go_left ? nd.left : nd.right;
}

// leaf values + output of the finished trees (one CTA per sequence), then the score update
__global__ void k_finish(GbdtState st, int iter) {
    const int s = blockIdx.x;
    const int n_nodes = st.n_nodes[s];
    Node* cur = st.cur + s * kMaxNodes;
    for (int nidx = threadIdx.x; nidx < n_nodes; nidx += blockDim.x) {
        if (cur[nidx].feature < 0) {
            const long long G = st.sumG[s * kMaxNodes + nidx], H = st.sumH[s * kMaxNodes + nidx];
            cur[nidx].value = H > 0 ? __dmul_rn(-__ddiv_rn((double)G, __dadd_rn((double)H, st.lam_q)), st.lr) : 0.0;
        }
        st.out[((size_t)iter * st.S + s) * kMaxNodes + nidx] = cur[nidx];
    }
    if (threadIdx.x == 0) st.out_count[iter * st.S + s] = n_nodes;
}

// k_finish with the options: L1 leaf -T(G) / (H + lambda_q), times lr_it (dart: lr / (1 + k)) or
// divided by n_iter (rf)
__global__ void k_finish_ex(GbdtState st, int iter, double lr_it) {
    const int s = blockIdx.x;
    const int n_nodes = st.n_nodes[s];
    Node* cur = st.cur + s * kMaxNodes;
    for (int nidx = threadIdx.x; nidx < n_nodes; nidx += blockDim.x) {
        if (cur[nidx].feature < 0) {
            const long long G = st.sumG[s * kMaxNodes + nidx], H = st.sumH[s * kMaxNodes + nidx];
            const double q = -__ddiv_rn(soft_q(G, st.alpha_q), __dadd_rn((double)H, st.lam_q));
            cur[nidx].value = H > 0 ? (st.rf_div > 0.0 ? __ddiv_rn(q, st.rf_div) : __dmul_rn(q, lr_it)) : 0.0;
        }
        st.out[((size_t)iter * st.S + s) * kMaxNodes + nidx] = cur[nidx];
    }
    if (threadIdx.x == 0) st.out_count[iter * st.S + s] = n_nodes;
}

// dart: scores[i][s] -= (add: +=) the leaf of row i in the finished trees (drops[j], s), j ascending
__global__ void __launch_bounds__(kThreads) k_dart_walk(GbdtState st, const int32_t* drops, int k, int add) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (i >= st.n) return;
    const uint8_t* row = st.bins + (size_t)i * st.F;
    double* sc = st.scores + (size_t)i * st.S + s;
    double v = *sc;
    for (int j = 0; j < k; ++j) {
        const Node* tree = st.out + ((size_t)drops[j] * st.S + s) * kMaxNodes;
        int nd = 0;
        while (tree[nd].feature >= 0) {
            const Node x = tree[nd];
            const int b = row[x.feature];
            const bool go_left = b == st.n_bins[x.feature] - 1 ? x.missing_left == 1 : b <= x.thr_bin;
            nd = go_left ? x.left : x.right;
        }
        v = add ? __dadd_rn(v, tree[nd].value) : __dsub_rn(v, tree[nd].value);
    }
    *sc = v;
}

// dart: the leaves of the dropped trees (CTA (j, s): tree (drops[j], s)) are multiplied by k / (k + 1)
__global__ void k_dart_scale(GbdtState st, const int32_t* drops, int k) {
    const int s = blockIdx.y;
    const size_t t = (size_t)drops[blockIdx.x] * st.S + s;
    Node* tree = st.out + t * kMaxNodes;
    const double f = __ddiv_rn((double)k, (double)(k + 1));
    for (int nidx = threadIdx.x; nidx < st.out_count[t]; nidx += blockDim.x)
        if (tree[nidx].feature < 0) tree[nidx].value = __dmul_rn(tree[nidx].value, f);
}

__global__ void __launch_bounds__(kThreads) k_update(GbdtState st) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (i >= st.n) return;
    const int node = st.node_of[(size_t)s * st.n + i];
    double* sc = st.scores + (size_t)i * st.S + s;
    *sc = __dadd_rn(*sc, st.cur[s * kMaxNodes + node].value);
}

__global__ void k_init_scores(GbdtState st, const double* init) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st.n) return;
    for (int s = 0; s < st.S; ++s) st.scores[(size_t)i * st.S + s] = init[s];
    st.inbag[i] = 1;
}

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

extern "C" {

int64_t dr_gbdt_workspace_bytes(int32_t n, int32_t n_seq) {
    size_t b = 0;
    b += align_up(sizeof(double) * (size_t)n * n_seq);          // scores
    b += 2 * align_up(sizeof(int32_t) * (size_t)n * n_seq);     // gq, hq
    b += align_up((size_t)n * n_seq);                           // node_of
    b += align_up((size_t)n);                                   // inbag
    b += 2 * align_up(sizeof(long long) * (size_t)n_seq * kMaxNodes);
    b += align_up(sizeof(int32_t) * (size_t)n_seq * kMaxNodes);
    b += align_up(sizeof(int32_t) * (size_t)n_seq * kMaxLeaves);
    b += 3 * align_up(sizeof(int32_t) * (size_t)n_seq);
    b += align_up(sizeof(Proposal) * (size_t)n_seq * kMaxLeaves);
    b += align_up(sizeof(Node) * (size_t)n_seq * kMaxNodes);
    b += align_up(sizeof(int32_t) * (size_t)n_seq * kMaxNodes);
    b += align_up(sizeof(double) * (size_t)n_seq);               // init
    return (int64_t)b;
}

int64_t dr_gbdt_train_ex_workspace_bytes(int32_t n, int32_t n_seq, int64_t n_drops) {
    size_t b = (size_t)dr_gbdt_workspace_bytes(n, n_seq);
    b += 2 * align_up(sizeof(double) * (size_t)n * n_seq);       // goss: g64, h64
    b += align_up(sizeof(double) * (size_t)n);                   // goss: row scores
    b += align_up(sizeof(unsigned long long));                   // goss: threshold bits
    b += align_up(sizeof(int32_t) * (size_t)(n_drops > 0 ? n_drops : 1));  // dart: dropped iterations
    return (int64_t)b;
}

int dr_gbdt_train_ex(dr_ctx* ctx, const dr_gbdt_params* prm, const dr_gbdt_boost* boost, const uint8_t* bins,
                     const int32_t* n_bins, const int32_t* y_class, const double* y_value, const double* weight,
                     const double* init, void* workspace, int64_t workspace_bytes, dr_gbdt_node* out_nodes,
                     int32_t* out_counts, void* stream) {
    if (!ctx) return DR_ERR_INVALID;
    DR_REQUIRE(ctx, prm && bins && n_bins && init && workspace && out_nodes && out_counts, "null pointer");
    static_assert(sizeof(Node) == sizeof(dr_gbdt_node), "node layout");
    const int n = prm->n_rows, F = prm->n_features;
    const int S = prm->n_classes <= 2 ? 1 : prm->n_classes;
    // the plain trainer unless some option is away from its default
    const bool plain = !boost || (boost->boosting == DR_GBDT_BOOST_GBDT && boost->reg_alpha == 0.0 &&
                                  boost->min_split_gain == 0.0);
    DR_REQUIRE(ctx, n > 0 && F > 0 && F <= 128, "n_rows > 0 and 1 <= n_features <= 128");
    DR_REQUIRE(ctx, prm->n_classes >= 1 && prm->n_iter >= 1, "bad n_classes / n_iter");
    DR_REQUIRE(ctx, prm->num_leaves >= 2 && prm->num_leaves <= kMaxLeaves, "num_leaves must be in [2, 32]");
    DR_REQUIRE(ctx, prm->max_depth >= 1 && prm->max_depth <= 31, "max_depth must be in [1, 31]");
    DR_REQUIRE(ctx, prm->n_classes == 1 ? y_value != nullptr : (y_class != nullptr && weight != nullptr),
               "missing targets / weights");
    const int boosting = plain ? DR_GBDT_BOOST_GBDT : boost->boosting;
    const bool dart = boosting == DR_GBDT_BOOST_DART, goss = boosting == DR_GBDT_BOOST_GOSS,
               rf = boosting == DR_GBDT_BOOST_RF;
    int64_t n_drops = 0;
    if (!plain) {
        DR_REQUIRE(ctx, boosting >= DR_GBDT_BOOST_GBDT && boosting <= DR_GBDT_BOOST_RF, "unknown boosting type");
        DR_REQUIRE(ctx, boost->reg_alpha >= 0.0 && boost->min_split_gain >= 0.0,
                   "reg_alpha and min_split_gain must be >= 0");
        if (dart) {
            DR_REQUIRE(ctx, boost->drop_off && boost->drop_off[0] == 0, "dart needs a drop schedule");
            for (int it = 0; it < prm->n_iter; ++it) {
                DR_REQUIRE(ctx, boost->drop_off[it + 1] >= boost->drop_off[it], "drop_off must not decrease");
                for (int j = boost->drop_off[it]; j < boost->drop_off[it + 1]; ++j)
                    DR_REQUIRE(ctx, boost->drop_iter && boost->drop_iter[j] >= 0 && boost->drop_iter[j] < it &&
                                        (j == boost->drop_off[it] || boost->drop_iter[j] > boost->drop_iter[j - 1]),
                               "an iteration drops earlier iterations, in ascending order");
            }
            n_drops = boost->drop_off[prm->n_iter];
        }
        if (goss)
            DR_REQUIRE(ctx, boost->goss_top_k >= 1 && boost->goss_top_k <= n && boost->goss_other_k >= 0 &&
                                boost->goss_other_k <= n - boost->goss_top_k && boost->goss_warmup >= 0,
                       "goss needs 1 <= top_k <= n_rows, 0 <= other_k <= n_rows - top_k and warmup >= 0");
        if (rf)
            DR_REQUIRE(ctx, (prm->subsample < 1.0 && prm->subsample_freq > 0) || prm->colsample_bytree < 1.0,
                       "boosting rf needs row bagging (subsample < 1 and subsample_freq > 0) or colsample_bytree < 1");
        DR_REQUIRE(ctx, workspace_bytes >= dr_gbdt_train_ex_workspace_bytes(n, S, n_drops), "workspace too small");
    } else {
        DR_REQUIRE(ctx, workspace_bytes >= dr_gbdt_workspace_bytes(n, S), "workspace too small");
    }
    DR_REQUIRE(ctx, prm->qscale > 0.0, "qscale must be positive");
    GbdtState st;
    memset(&st, 0, sizeof(st));
    st.bins = bins; st.y_class = y_class; st.y_value = y_value; st.weight = weight;
    st.n = n; st.F = F; st.S = S; st.n_classes = prm->n_classes; st.max_depth = prm->max_depth;
    st.num_leaves = prm->num_leaves; st.min_data = prm->min_data_in_leaf;
    st.lr = prm->learning_rate; st.qscale = prm->qscale; st.min_hess_q = prm->min_sum_hessian * prm->qscale;
    st.factor = S > 1 ? (double)S / (double)(S - 1) : 1.0;
    DR_REQUIRE(ctx, prm->reg_lambda >= 0.0, "reg_lambda must be >= 0");
    DR_REQUIRE(ctx, prm->colsample_bytree > 0.0 && prm->subsample > 0.0, "sampling fractions must be positive");
    st.lam_q = prm->reg_lambda * prm->qscale;
    st.col_thr = prm->colsample_bytree >= 1.0 ? -1 : (int)(prm->colsample_bytree * 16777216.0);
    const bool bagging = prm->subsample < 1.0 && prm->subsample_freq > 0 && !goss;  // goss ignores bagging
    st.bag_freq = bagging ? prm->subsample_freq : 0;
    st.bag_thr = bagging ? (int)(prm->subsample * 16777216.0) : 0;
    st.seed = (unsigned long long)(long long)prm->seed;
    int total = 0;
    for (int f = 0; f < F; ++f) {
        DR_REQUIRE(ctx, n_bins[f] >= 1 && n_bins[f] <= 256, "bins per feature must be in [1, 256]");
        st.n_bins[f] = n_bins[f];
        st.bin_off[f] = total;
        total += n_bins[f];
    }
    st.bin_off[F] = total;
    const size_t smem = (size_t)total * 12;
    if (smem > 200 * 1024)
        return dr_fail(ctx, DR_ERR_UNSUPPORTED, "%d histogram bins do not fit in shared memory", total);
    unsigned char* w = (unsigned char*)workspace;
    auto take = [&](size_t bytes) { void* p = w; w += align_up(bytes); return p; };
    st.scores = (double*)take(sizeof(double) * (size_t)n * S);
    st.gq = (int32_t*)take(sizeof(int32_t) * (size_t)n * S);
    st.hq = (int32_t*)take(sizeof(int32_t) * (size_t)n * S);
    st.node_of = (uint8_t*)take((size_t)n * S);
    st.inbag = (uint8_t*)take((size_t)n);
    st.sumG = (long long*)take(sizeof(long long) * (size_t)S * kMaxNodes);
    st.sumH = (long long*)take(sizeof(long long) * (size_t)S * kMaxNodes);
    st.sumC = (int32_t*)take(sizeof(int32_t) * (size_t)S * kMaxNodes);
    st.active = (int32_t*)take(sizeof(int32_t) * (size_t)S * kMaxLeaves);
    st.n_active = (int32_t*)take(sizeof(int32_t) * (size_t)S);
    st.n_nodes = (int32_t*)take(sizeof(int32_t) * (size_t)S);
    st.n_leaves = (int32_t*)take(sizeof(int32_t) * (size_t)S);
    st.props = (Proposal*)take(sizeof(Proposal) * (size_t)S * kMaxLeaves);
    st.cur = (Node*)take(sizeof(Node) * (size_t)S * kMaxNodes);
    st.split_flag = (int32_t*)take(sizeof(int32_t) * (size_t)S * kMaxNodes);
    double* d_init = (double*)take(sizeof(double) * (size_t)S);
    st.out = reinterpret_cast<Node*>(out_nodes);
    st.out_count = out_counts;
    cudaStream_t sm = (cudaStream_t)stream;
    DR_CUDA(ctx, cudaMemcpyAsync(d_init, init, sizeof(double) * S, cudaMemcpyHostToDevice, sm));
    const int row_blocks = (n + kThreads - 1) / kThreads;
    if (plain) {
        DR_CUDA(ctx, cudaFuncSetAttribute(k_level<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_init_scores<<<row_blocks, kThreads, 0, sm>>>(st, d_init);
        DR_LAUNCHED(ctx);
        for (int it = 0; it < prm->n_iter; ++it) {
            k_grad<<<row_blocks, kThreads, 0, sm>>>(st, it);
            k_root<<<S, kThreads, 0, sm>>>(st);
            for (int depth = 0; depth < prm->max_depth; ++depth) {
                k_level<false><<<dim3(S, kMaxLeaves), kThreads, smem, sm>>>(st, it);
                k_apply<<<(S + 63) / 64, 64, 0, sm>>>(st, depth);
                k_reassign<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st);
            }
            k_finish<<<S, 64, 0, sm>>>(st, it);
            k_update<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st);
            ctx->launches += 3 + 3 * prm->max_depth;
        }
        DR_CUDA(ctx, cudaGetLastError());
        return DR_OK;
    }
    // ---- with boosting options (oracle/gbdt_boost.py) ----
    st.alpha_q = boost->reg_alpha * prm->qscale;
    st.gain_floor = boost->min_split_gain * prm->qscale;
    st.rf_div = rf ? (double)prm->n_iter : 0.0;
    st.g64 = (double*)take(sizeof(double) * (size_t)n * S);
    st.h64 = (double*)take(sizeof(double) * (size_t)n * S);
    st.rscore = (double*)take(sizeof(double) * (size_t)n);
    st.goss_tau = (unsigned long long*)take(sizeof(unsigned long long));
    int32_t* d_drops = (int32_t*)take(sizeof(int32_t) * (size_t)(n_drops > 0 ? n_drops : 1));
    if (goss) {
        const int top_k = boost->goss_top_k, other_k = boost->goss_other_k;
        st.goss_top_k = top_k;
        st.goss_amp = other_k > 0 ? (double)(n - top_k) / (double)other_k : 1.0;
        st.goss_other_thr = n > top_k ? (int)((double)other_k / (double)(n - top_k) * 16777216.0) : 0;
    }
    if (n_drops > 0)
        DR_CUDA(ctx, cudaMemcpyAsync(d_drops, boost->drop_iter, sizeof(int32_t) * (size_t)n_drops,
                                     cudaMemcpyHostToDevice, sm));
    DR_CUDA(ctx, cudaFuncSetAttribute(k_level<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_init_scores<<<row_blocks, kThreads, 0, sm>>>(st, d_init);
    DR_LAUNCHED(ctx);
    for (int it = 0; it < prm->n_iter; ++it) {
        const int k = dart ? boost->drop_off[it + 1] - boost->drop_off[it] : 0;
        const int32_t* drops = d_drops + (dart ? boost->drop_off[it] : 0);
        if (k > 0) {  // the dropped trees leave the scores
            k_dart_walk<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st, drops, k, 0);
            ctx->launches += 1;
        }
        if (rf && it > 0) {
            k_bag<<<row_blocks, kThreads, 0, sm>>>(st, it);
            ctx->launches += 1;
        } else if (goss && it >= boost->goss_warmup) {
            k_grad64<<<row_blocks, kThreads, 0, sm>>>(st);
            k_goss_select<<<1, kSelectThreads, 0, sm>>>(st);
            k_goss_apply<<<row_blocks, kThreads, 0, sm>>>(st, it);
            ctx->launches += 3;
        } else {
            k_grad<<<row_blocks, kThreads, 0, sm>>>(st, it);
            ctx->launches += 1;
        }
        k_root<<<S, kThreads, 0, sm>>>(st);
        for (int depth = 0; depth < prm->max_depth; ++depth) {
            k_level<true><<<dim3(S, kMaxLeaves), kThreads, smem, sm>>>(st, it);
            k_apply<<<(S + 63) / 64, 64, 0, sm>>>(st, depth);
            k_reassign<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st);
        }
        k_finish_ex<<<S, 64, 0, sm>>>(st, it, prm->learning_rate / (1.0 + k));
        ctx->launches += 2 + 3 * prm->max_depth;
        if (!rf) {
            k_update<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st);
            ctx->launches += 1;
        }
        if (k > 0) {  // and return rescaled
            k_dart_scale<<<dim3(k, S), 64, 0, sm>>>(st, drops, k);
            k_dart_walk<<<dim3(row_blocks, S), kThreads, 0, sm>>>(st, drops, k, 1);
            ctx->launches += 2;
        }
    }
    DR_CUDA(ctx, cudaGetLastError());
    return DR_OK;
}

int dr_gbdt_train(dr_ctx* ctx, const dr_gbdt_params* prm, const uint8_t* bins, const int32_t* n_bins,
                  const int32_t* y_class, const double* y_value, const double* weight, const double* init,
                  void* workspace, int64_t workspace_bytes, dr_gbdt_node* out_nodes, int32_t* out_counts,
                  void* stream) {
    return dr_gbdt_train_ex(ctx, prm, nullptr, bins, n_bins, y_class, y_value, weight, init, workspace,
                            workspace_bytes, out_nodes, out_counts, stream);
}

}  // extern "C"
