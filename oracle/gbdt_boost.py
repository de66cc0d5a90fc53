"""Oracle of the GPU trainer's boosting options (TEST INFRASTRUCTURE -- see oracle/__init__.py).

``train()`` is ``oracle/gbdt.py``'s trainer with the ``model.lgb.*`` options the reference hands to
LightGBM 3.3.1 (``train.py:102-115``) and the plain trainer does not take: ``boosting`` (gbdt, dart,
goss, rf), ``reg_alpha`` and ``min_split_gain``.  At their defaults it performs exactly the operations
of ``oracle/gbdt.py`` (``tests/test_gbdt_options_cpu.py`` pins the hashes of its forests).
The GOSS and DART constants (``top_rate`` 0.2, ``other_rate`` 0.1, ``drop_rate`` 0.1, ``max_drop`` 50,
``skip_drop`` 0.5) are LightGBM 3.3.1's documented defaults; the reference does not expose them.
LightGBM is not installed, so these semantics are RESTATED from its documentation and sources, not
pinned against it.  Everything happens in the quantised integer space of ``oracle/gbdt.py``; every
random draw is a splitmix64 hash (``mix64``), as the feature subsets and row bags already are.

* reg_alpha (L1): with a_q = reg_alpha * qscale and T(G) = sign(G) * max(|G| - a_q, 0), gains use
  T(G)^2 / (H + lambda_q) and leaves -T(G) / (H + lambda_q) * learning rate.
* min_split_gain: a leaf's best split is proposed only when its gain > min_split_gain * qscale.
* goss: no sampling for the first int(1 / learning_rate) iterations.  Then row i's score is
  sum over classes (ascending) of |g * h| (unquantised float64); rows whose score is >= the top_k-th
  largest (top_k = max(1, int(n * top_rate))) are kept, ties included; every other row is kept iff
  hash(seed, iteration, i) < other_k / (n - top_k) (other_k = int(n * other_rate)), its g and h
  multiplied by m = (n - top_k) / other_k before quantisation.  qscale is divided by 2^ceil(log2 m)
  for the whole run, so histograms still fit int32.  goss ignores subsample / subsample_freq.
* rf: gradients and hessians once, at the initial scores; every iteration draws its bag and feature
  subset as gbdt does; leaf value -T(G) / (H + lambda_q) / n_iter, so baseline + sum of leaves is the
  average of the trees.  Needs row bagging or colsample_bytree < 1 (LightGBM refuses rf otherwise).
* dart: the drop schedule (``dart_schedule``) depends only on iteration numbers and tree weights.
  A new tree's shrinkage is learning_rate / (1 + k) for k dropped iterations, then the dropped trees'
  leaves and weights are multiplied by k / (k + 1).  Per (row, class) the score updates are: subtract
  the dropped trees (ascending iteration), train, add the new tree, add the rescaled dropped trees
  (ascending).  The initial score stays outside the trees and is never dropped (LightGBM folds it
  into its first tree).
"""
import numpy as np

from .gbdt import (feature_used, mix64, quant_bits, rows_in_bag, sigmoid_det, softmax_det,  # noqa: F401
                   to_flat_forest)

BOOSTING = ("gbdt", "dart", "goss", "rf")
_GOLDEN = 0x9E3779B97F4A7C15


def _h24(key):
    return mix64(key) >> 40


def ceil_log2(m):
    """Smallest e >= 0 with 2^e >= m."""
    e = 0
    while float(1 << e) < m:
        e += 1
    return e


def goss_counts(n, top_rate=0.2, other_rate=0.1):
    """-> (top_k, other_k, m, qscale shift) of GOSS on n rows."""
    top_k, other_k = max(1, int(n * top_rate)), int(n * other_rate)
    m = (n - top_k) / other_k if other_k > 0 else 1.0
    return top_k, other_k, m, ceil_log2(m)


def goss_other_thr(n, top_k, other_k):
    """24-bit threshold of the draw that keeps a non-top row."""
    return int(other_k / (n - top_k) * float(1 << 24)) if n > top_k else 0


def goss_hash(seed, it, n):
    return np.array([_h24((seed + 2) * _GOLDEN + (it << 32) + i) for i in range(n)], dtype=np.int64)


def goss_rows(g, h, seed, it, top_k, other_thr):
    """-> (kept bool[n], top bool[n]) of GOSS iteration it from float64 g, h [n, S]."""
    score = np.zeros(len(g))
    for s in range(g.shape[1]):                    # ascending class
        score = score + np.abs(g[:, s] * h[:, s])
    tau = np.sort(score)[::-1][top_k - 1]
    top = score >= tau
    return top | (goss_hash(seed, it, len(g)) < other_thr), top


def dart_schedule(n_iter, learning_rate, seed, drop_rate=0.1, max_drop=50, skip_drop=0.5):
    """-> list over iterations of the earlier iterations it drops (ascending).

    Iteration it skips dropping iff hash(seed, it) / 2^24 < skip_drop.  Otherwise earlier iteration i is
    dropped iff hash(seed, it, i) / 2^24 < rate * w_i * T / W (T = it trees so far, W = sum of their
    weights w, rate = min(drop_rate, max_drop * (T / W) / W): LightGBM's non-uniform rule), up to max_drop
    drops.  Then W -= w_i / (k + 1) and w_i *= k / (k + 1) per dropped i, and the new tree's weight is its
    shrinkage learning_rate / (1 + k)."""
    weights, total, out = [], 0.0, []
    for it in range(n_iter):
        drops = []
        if it > 0 and not (_h24((seed + 4) * _GOLDEN + it) / float(1 << 24) < skip_drop):
            inv_avg = float(it) / total
            rate = drop_rate
            if max_drop > 0:
                rate = min(rate, max_drop * inv_avg / total)
            for i in range(it):
                if _h24((seed + 3) * _GOLDEN + (it << 32) + i) / float(1 << 24) < rate * weights[i] * inv_avg:
                    drops.append(i)
                    if max_drop > 0 and len(drops) >= max_drop:
                        break
        k = len(drops)
        for i in drops:
            total -= weights[i] * (1.0 / (k + 1.0))
            weights[i] *= k / (k + 1.0)
        shrink = learning_rate / (1.0 + k)
        weights.append(shrink)
        total += shrink
        out.append(drops)
    return out


def leaf_of(nodes, bins, n_bins):
    """int64[n]: the node every row of bins reaches in one tree (node lists as train() returns them)."""
    node = np.zeros(len(bins), dtype=np.int64)
    while True:
        feat = np.array([nodes[j][0] for j in node])
        inner = feat >= 0
        if not inner.any():
            return node
        for j in np.unique(node[inner]):
            f, t, ml, l, r, _ = nodes[j]
            rows = np.nonzero(node == j)[0]
            b = bins[rows, f].astype(np.int64)
            go_left = np.where(b == n_bins[f] - 1, ml == 1, b <= t)
            node[rows] = np.where(go_left, l, r)


def train(bins, n_bins, y, n_classes, sample_weight=None, n_iter=300, learning_rate=0.01, max_depth=7,
          num_leaves=31, min_data_in_leaf=20, min_sum_hessian=1e-3, reg_lambda=0.0, colsample_bytree=1.0,
          subsample=1.0, subsample_freq=0, seed=42, boosting="gbdt", reg_alpha=0.0, min_split_gain=0.0,
          top_rate=0.2, other_rate=0.1, drop_rate=0.1, max_drop=50, skip_drop=0.5, quant_shift=None):
    """oracle/gbdt.py train() plus the boosting options (module docstring).  quant_shift: extra right
    shift of the quantisation scale (None: goss's ceil(log2 m) under goss, else 0)."""
    if boosting not in BOOSTING:
        raise ValueError("boosting must be one of {}".format(BOOSTING))
    bins = np.asarray(bins)
    n, F = bins.shape
    S = 1 if n_classes <= 2 else n_classes
    w = np.ones(n) if sample_weight is None else np.asarray(sample_weight, dtype=np.float64)
    qscale = float(2 ** quant_bits(n)) / float(w.max())
    scores = np.zeros((n, S))
    if n_classes == 1:
        yv = np.asarray(y, dtype=np.float64)
        init = np.array([np.cumsum(yv)[-1] / n])  # sequential sum
        qscale = float(2 ** quant_bits(n)) / max(float(np.abs(yv - init[0]).max()), 1e-300)
    elif n_classes == 2:
        yv = np.asarray(y, dtype=np.float64)
        sw, swy = np.cumsum(w)[-1], np.cumsum(w * yv)[-1]  # sequential sums
        pavg = min(max(swy / sw, 1e-15), 1.0 - 1e-15)
        init = np.array([np.log(pavg / (1.0 - pavg))])
    else:
        init = np.zeros(S)
        onehot = np.zeros((n, S))
        onehot[np.arange(n), np.asarray(y, dtype=np.int64)] = 1.0
    scores += init[None, :]
    goss = boosting == "goss"
    if goss:
        top_k, other_k, amp, shift = goss_counts(n, top_rate, other_rate)
        other_thr = goss_other_thr(n, top_k, other_k)
        warmup = int(1.0 / learning_rate)
    else:
        shift = 0
    if quant_shift is not None:
        shift = quant_shift
    qscale = qscale / float(1 << shift)
    offs = np.zeros(F + 1, dtype=np.int64)
    offs[1:] = np.cumsum(n_bins)
    flat = bins.astype(np.int64) + offs[:-1][None, :]      # [n, F] global bin ids
    trees = []
    lam_q = float(reg_lambda) * qscale
    alpha_q = float(reg_alpha) * qscale
    floor = float(min_split_gain) * qscale
    bagging = subsample < 1.0 and subsample_freq > 0 and not goss
    if boosting == "rf" and not (bagging or colsample_bytree < 1.0):
        raise ValueError("boosting rf needs row bagging (subsample < 1 and subsample_freq > 0) "
                         "or colsample_bytree < 1")
    schedule = dart_schedule(n_iter, learning_rate, seed, drop_rate, max_drop, skip_drop) \
        if boosting == "dart" else [[]] * n_iter

    def soft(G):  # T(G); at reg_alpha = 0 the plain trainer's float(G)
        if alpha_q == 0.0:
            return float(G)
        a = abs(float(G)) - alpha_q
        return 0.0 if not a > 0.0 else (a if G > 0 else -a)

    def gain_term(G, H):
        if alpha_q == 0.0:
            return (float(G) * float(G)) / (float(H) + lam_q)
        t = soft(G)
        return (t * t) / (float(H) + lam_q)

    in_bag = np.ones(n, dtype=bool)
    for it in range(n_iter):
        drops = schedule[it]
        for d in drops:                            # 1. the dropped trees leave the scores
            for s in range(S):
                nodes = trees[d][s]
                scores[:, s] = scores[:, s] - np.array([nd[5] for nd in nodes])[leaf_of(nodes, bins, n_bins)]
        if bagging and it % subsample_freq == 0:
            in_bag = rows_in_bag(seed, it // subsample_freq, n, subsample)
        if boosting != "rf" or it == 0:
            if n_classes == 1:
                g, h = scores - yv[:, None], np.ones((n, 1))
            elif n_classes == 2:
                p = sigmoid_det(scores[:, 0])
                g, h = ((p - yv) * w)[:, None], (p * (1.0 - p) * w)[:, None]
            else:
                p = softmax_det(scores)
                factor = float(S) / float(S - 1)
                g, h = (p - onehot) * w[:, None], factor * p * (1.0 - p) * w[:, None]
            if goss and it >= warmup:
                in_bag, top = goss_rows(g, h, seed, it, top_k, other_thr)
                g = np.where(top[:, None], g, g * amp)
                h = np.where(top[:, None], h, h * amp)
            gq, hq = np.rint(g * qscale).astype(np.int64), np.rint(h * qscale).astype(np.int64)
        lr_it = learning_rate / (1.0 + len(drops)) if drops else learning_rate
        it_trees = []
        for s in range(S):
            nodes = [[-1, 0, 0, 0, 0, 0.0]]
            node_of = np.zeros(n, dtype=np.int64)
            used = feature_used(seed, it, s, F, colsample_bytree)
            sums = {0: (int(gq[in_bag, s].sum()), int(hq[in_bag, s].sum()), int(in_bag.sum()))}
            active, n_leaves = [0], 1
            for depth in range(max_depth):
                props = []
                for leaf in active:
                    rows = np.nonzero((node_of == leaf) & in_bag)[0]
                    G, H, cnt = sums[leaf]
                    if cnt < 2 * min_data_in_leaf or H <= 0:
                        continue
                    idx = flat[rows].reshape(-1)
                    hg = np.zeros(offs[-1], dtype=np.int64)
                    hh = np.zeros(offs[-1], dtype=np.int64)
                    hc = np.zeros(offs[-1], dtype=np.int64)
                    np.add.at(hg, idx, np.repeat(gq[rows, s], F))
                    np.add.at(hh, idx, np.repeat(hq[rows, s], F))
                    np.add.at(hc, idx, 1)
                    best = None
                    parent = gain_term(G, H)
                    for f in range(F):
                        nb = int(n_bins[f])
                        if nb < 3 or not used[f]:
                            continue
                        o = int(offs[f])
                        mg, mh, mc = int(hg[o + nb - 1]), int(hh[o + nb - 1]), int(hc[o + nb - 1])
                        cg = ch = cc = 0
                        for t in range(nb - 2):  # split after value bin t
                            cg += int(hg[o + t]); ch += int(hh[o + t]); cc += int(hc[o + t])
                            for ml in (0, 1):
                                GL, HL, CL = (cg + mg, ch + mh, cc + mc) if ml else (cg, ch, cc)
                                GR, HR, CR = G - GL, H - HL, cnt - CL
                                if CL < min_data_in_leaf or CR < min_data_in_leaf:
                                    continue
                                if HL < min_sum_hessian * qscale or HR < min_sum_hessian * qscale:
                                    continue
                                gain = (gain_term(GL, HL) + gain_term(GR, HR)) - parent
                                if gain > 0.0 and (best is None or gain > best[0]):
                                    best = (gain, f, t, ml, GL, HL, CL)
                    if best is not None and best[0] > floor:
                        props.append((best, leaf))
                props.sort(key=lambda pr: (-pr[0][0], pr[1]))
                new_active = []
                for (gain, f, t, ml, GL, HL, CL), leaf in props:
                    if n_leaves >= num_leaves:
                        break
                    G, H, cnt = sums[leaf]
                    li, ri = len(nodes), len(nodes) + 1
                    nodes[leaf][0:5] = [f, t, ml, li, ri]
                    nodes += [[-1, 0, 0, 0, 0, 0.0], [-1, 0, 0, 0, 0, 0.0]]
                    sums[li], sums[ri] = (GL, HL, CL), (G - GL, H - HL, cnt - CL)
                    rows = np.nonzero(node_of == leaf)[0]
                    b = bins[rows, f].astype(np.int64)
                    go_left = np.where(b == n_bins[f] - 1, ml == 1, b <= t)
                    node_of[rows] = np.where(go_left, li, ri)
                    new_active += [li, ri]
                    n_leaves += 1
                active = new_active
                if not active:
                    break
            for i, nd in enumerate(nodes):
                if nd[0] < 0:
                    G, H, _ = sums[i]
                    if not H > 0:
                        nd[5] = 0.0
                    elif boosting == "rf":
                        nd[5] = (-(soft(G) / (float(H) + lam_q))) / float(n_iter)
                    else:
                        nd[5] = (-(soft(G) / (float(H) + lam_q))) * lr_it
            vals = np.array([nd[5] for nd in nodes])
            if boosting != "rf":
                scores[:, s] = scores[:, s] + vals[node_of]  # 3. the new tree
            it_trees.append([tuple(nd) for nd in nodes])
        trees.append(it_trees)
        if drops:                                  # 4. the dropped trees return, rescaled
            k = len(drops)
            scale = float(k) / float(k + 1)
            for d in drops:
                trees[d] = [[(f, t, ml, l, r, v * scale if f < 0 else v) for (f, t, ml, l, r, v) in nodes]
                            for nodes in trees[d]]
            for d in drops:
                for s in range(S):
                    nodes = trees[d][s]
                    scores[:, s] = scores[:, s] + np.array([nd[5] for nd in nodes])[leaf_of(nodes, bins, n_bins)]
    return {"init": init, "trees": trees, "n_classes": n_classes}
