"""GPU histogram-GBDT trainer (host side of ``dr_gbdt_train``): pre-bins the encoded training
sample, computes class weights / initial scores, runs the whole boosting loop on the device and
flattens the result into the exchange format of ``forest.py``.

Eligibility: at most 128 encoded features; a feature with more than max_bin - 1 distinct values (254 at
the default max_bin = 255) is binned like LightGBM's max_bin does (adjacent values share a bin).  Which
models come here is decided by ``model.gpu_trainer_bins``: every all-discrete model, and models with a
continuous target or feature when a boosting option is set; the others use ``train.build_model``
(scikit-learn).

Boosting options (``model.lgb.boosting_type`` dart / goss / rf, ``reg_alpha``, ``min_split_gain``) run
through ``dr_gbdt_train_ex``; at their defaults the trainer is called exactly as before."""
import math

import numpy as np

from .forest import encoder_lut

NODE_DTYPE = np.dtype([("feature", np.int16), ("thr_bin", np.uint8), ("missing_left", np.uint8), ("left", np.uint8),
                       ("right", np.uint8), ("pad", np.uint8, (2,)), ("value", np.float64)])
MAX_NODES = 64
MAX_BINS = 254   # real bins per feature (one more is the missing bin; bins travel as bytes)


def quant_bits(n_rows):
    """Quantisation width: every histogram bin (a sum over <= n_rows rows) must fit a signed 32-bit
    integer, so that the device can use native 32-bit shared-memory atomics."""
    return int(min(24, 30 - int(np.ceil(np.log2(max(n_rows, 2))))))


def bin_column(x, domain, max_real):
    """One encoded feature -> (bins uint8 [n], n_bins, bin values).  x: the sample's float64 values (NaN =
    NULL, which goes to the missing bin n_bins - 1); domain: the sorted distinct values the feature can
    take (never NaN).  Up to max_real distinct values: one bin per value, bin values 1-D.  More: adjacent
    values share a bin (LightGBM: max_bin = 255, train.py:106), bins of about equal sample counts, bin
    values 2 x n_real (largest / smallest value of every bin); thresholds only fall between bins."""
    ok = ~np.isnan(x)
    pos = np.searchsorted(domain, x[ok])
    if len(domain) > max_real:
        cnt = np.bincount(pos, minlength=len(domain)).astype(np.float64)
        edge = np.floor(np.cumsum(cnt) / max(cnt.sum(), 1.0) * max_real - 1e-9).astype(np.int64)
        group = np.minimum(np.maximum.accumulate(np.clip(edge, 0, max_real - 1)), max_real - 1)
        _, group = np.unique(group, return_inverse=True)      # dense bin ids, in value order
        n_real = int(group.max()) + 1
        values = np.stack([np.array([domain[group == b].max() for b in range(n_real)]),
                           np.array([domain[group == b].min() for b in range(n_real)])])
    else:
        group, n_real, values = np.arange(len(domain)), len(domain), domain
    out = np.full(len(x), n_real, dtype=np.uint8)                          # missing bin
    out[ok] = group[pos].astype(np.uint8)
    return out, n_real + 1, values


def bin_sample(encoders, sample_codes, dict_sizes, max_bin=255, sample_values=None):
    """-> (bins uint8 [n, F'], n_bins int32 [F'], bin_values list of float arrays) or None.
    A feature gets at most max_bin - 1 value bins (max_bin clamped to [2, 255]) plus the missing bin.
    A discrete feature's domain is every value its encoder LUT holds; a continuous one ("cont" encoder,
    float64 column of sample_values = {attr: values}, NaN = NULL) takes the sample's distinct values, +-inf
    included, so an all-NULL column has only the missing bin and a single-valued one two bins.  None when
    a continuous feature's values are not given or there are more than 128 encoded features."""
    max_real = min(255, max(2, int(max_bin))) - 1
    cols, n_bins, values = [], [], []
    for e in encoders:
        if e["type"] == "cont":
            if sample_values is None or e["attr"] not in sample_values:
                return None
            x = np.asarray(sample_values[e["attr"]], dtype=np.float64)
            parts = [bin_column(x, np.unique(x[~np.isnan(x)]), max_real)]
        else:
            lut = encoder_lut(e, dict_sizes[e["attr"]])
            codes = np.asarray(sample_codes[e["attr"]], dtype=np.int64)
            parts = [bin_column(lut[codes + 1, j], np.unique(lut[~np.isnan(lut[:, j]), j]), max_real)
                     for j in range(lut.shape[1])]
        for b, nb, v in parts:
            cols.append(b)
            n_bins.append(nb)
            values.append(v)
    if not cols or len(cols) > 128:
        return None
    return np.stack(cols, axis=1).astype(np.uint8), np.asarray(n_bins, dtype=np.int32), values


MIN_HESS_QUANTUM = 1024.0   # a regression row's quantised hessian: rounding bias <= 0.5 / 1024 of every leaf


def regression_scale(y, init, n, goss_shift=0):
    """-> k: a regression trains on y * 2^-k and its leaves and baseline are multiplied back by 2^k.
    Every row's hessian 1 is quantised as the scale itself, 2^bits / max|y - init| / 2^goss_shift.  A spread
    below 1 would push the hessian sums past int32; a large one (prices, incomes) rounds the hessian to a few
    units or to 0, which biases every leaf or leaves the trees without a split.  So outside 1 <= spread with a
    quantum >= MIN_HESS_QUANTUM, the target is brought to a spread in [1, 2), a quantum of at least
    2^(bits - 1 - goss_shift).  Scaling by a power of two is exact, and with reg_alpha * 2^-k and min_split_gain
    * 2^-2k every leaf of the scaled problem is the original's times 2^-k and every gain times 2^-2k in exact
    arithmetic, so only the fineness of the quantisation changes.  Inside the window k = 0: the trainer runs
    exactly as oracle/gbdt.py specifies it on the unscaled target."""
    spread = float(np.abs(np.asarray(y, dtype=np.float64) - init).max())
    if not spread > 0.0 or not np.isfinite(spread):
        return 0
    quantum = float(2 ** quant_bits(n)) / spread / float(1 << goss_shift)
    if spread >= 1.0 and quantum >= MIN_HESS_QUANTUM:
        return 0
    return math.frexp(spread)[1] - 1          # spread = m * 2^e, m in [0.5, 1): spread * 2^-(e-1) in [1, 2)


def class_weights(y_idx, n_classes, balanced):
    """class_weight='balanced' (train.py:105): n / (C * count[class])."""
    n = len(y_idx)
    if not balanced:
        return np.ones(n)
    cnt = np.bincount(y_idx, minlength=n_classes).astype(np.float64)
    return (float(n) / (float(n_classes) * cnt))[y_idx]


def initial_scores(y, n_classes, weight):
    if n_classes == 1:
        yv = np.asarray(y, dtype=np.float64)
        return np.array([np.cumsum(yv)[-1] / len(yv)])
    if n_classes == 2:
        yv = np.asarray(y, dtype=np.float64)
        sw, swy = np.cumsum(weight)[-1], np.cumsum(weight * yv)[-1]
        pavg = min(max(swy / sw, 1e-15), 1.0 - 1e-15)
        return np.array([np.log(pavg / (1.0 - pavg))])
    return np.zeros(n_classes)


def _h24(key):
    """Top 24 bits of the splitmix64 finaliser of key (the trainer's hash)."""
    z = key & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return (z ^ (z >> 31)) >> 40


_M64 = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15


def dart_schedule(n_iter, learning_rate, seed, drop_rate=0.1, max_drop=50, skip_drop=0.5):
    """DART's drop schedule -> (drop_off int32 [n_iter + 1], drop_iter int32): iteration it drops the earlier
    iterations drop_iter[drop_off[it]:drop_off[it + 1]].  LightGBM's non-uniform rule over tree weights:
    an iteration skips dropping with probability skip_drop; otherwise tree i goes with probability
    rate * w_i * T / W (T trees of total weight W, rate = min(drop_rate, max_drop * T / W^2)), at most
    max_drop of them; a new tree weighs learning_rate / (1 + k), dropped ones shrink by k / (k + 1)."""
    unit = float(1 << 24)
    weights, total = [], 0.0
    off, flat = [0], []
    for it in range(n_iter):
        k = 0
        if it > 0 and _h24((seed + 4) * _GOLDEN + it) / unit >= skip_drop:
            inv_avg = float(it) / total
            rate = min(drop_rate, max_drop * inv_avg / total) if max_drop > 0 else drop_rate
            for i in range(it):
                if _h24((seed + 3) * _GOLDEN + (it << 32) + i) / unit < rate * weights[i] * inv_avg:
                    flat.append(i)
                    k += 1
                    if k == max_drop:
                        break
        for i in flat[len(flat) - k:]:
            total -= weights[i] * (1.0 / (k + 1.0))
            weights[i] *= k / (k + 1.0)
        weights.append(learning_rate / (1.0 + k))
        total += weights[-1]
        off.append(len(flat))
    return np.asarray(off, dtype=np.int32), np.asarray(flat, dtype=np.int32)


def goss_counts(n, top_rate=0.2, other_rate=0.1):
    """-> (top_k, other_k, quantisation shift): GOSS keeps the top_k rows by |g * h| and draws the others
    with probability other_k / (n - top_k), amplified by m = (n - top_k) / other_k; qscale is divided by
    2^ceil(log2 m) so that histogram bins keep fitting int32."""
    top_k, other_k = max(1, int(n * top_rate)), int(n * other_rate)
    m = (n - top_k) / other_k if other_k > 0 else 1.0
    shift = 0
    while float(1 << shift) < m:
        shift += 1
    return top_k, other_k, shift


def train_gpu(ctx, device, bins, n_bins, bin_values, y, n_classes, weight, n_iter, learning_rate, max_depth,
              num_leaves=31, min_data_in_leaf=20, min_sum_hessian=1e-3, reg_lambda=0.0, colsample_bytree=1.0,
              subsample=1.0, subsample_freq=0, seed=42, boosting="gbdt", reg_alpha=0.0, min_split_gain=0.0,
              top_rate=0.2, other_rate=0.1, drop_rate=0.1, max_drop=50, skip_drop=0.5):
    """-> flat forest (forest.py layout).  boosting / reg_alpha / min_split_gain away from their defaults
    select dr_gbdt_train_ex (top_rate / other_rate: goss, drop_rate / max_drop / skip_drop: dart)."""
    import torch
    from ._native import DR_GBDT_BOOST, dr_gbdt_boost, dr_gbdt_params
    if boosting not in DR_GBDT_BOOST:
        raise ValueError("boosting must be one of {}".format(sorted(DR_GBDT_BOOST)))
    # the device indexes its shared-memory histograms with every bin byte: check them all before any launch
    n_bins = np.asarray(n_bins, dtype=np.int32)
    if bins.dtype != np.uint8 or bins.ndim != 2 or bins.shape[1] != len(n_bins):
        raise ValueError("bins must be uint8 [n, {}] (one column per n_bins entry), got {} {}".format(
            len(n_bins), bins.dtype, bins.shape))
    if len(n_bins) and (int(n_bins.min()) < 1 or int(n_bins.max()) > 255):
        raise ValueError("bins per feature must be in [1, 255]")
    if bins.size and (bins >= n_bins).any():
        f = int(np.flatnonzero((bins >= n_bins).any(axis=0))[0])
        raise ValueError("feature {}: bin byte {} >= n_bins {}".format(f, int(bins[:, f].max()), int(n_bins[f])))
    n, F = bins.shape
    S = 1 if n_classes <= 2 else n_classes
    top_k, other_k, goss_shift = goss_counts(n, top_rate, other_rate) if boosting == "goss" else (0, 0, 0)
    k = 0
    if n_classes == 1:
        y = np.asarray(y, dtype=np.float64)
        k = regression_scale(y, initial_scores(y, 1, None)[0], n, goss_shift)
        y = np.ldexp(y, -k)
        reg_alpha, min_split_gain = float(np.ldexp(reg_alpha, -k)), float(np.ldexp(min_split_gain, -2 * k))
    init = initial_scores(y, n_classes, weight)
    if n_classes == 1:
        spread = float(np.abs(y - init[0]).max())
        qscale = float(2 ** quant_bits(n)) / (spread if spread > 0.0 else 1.0)   # constant target: any scale
    else:
        qscale = float(2 ** quant_bits(n)) / float(np.max(weight))
    boost = None
    if boosting != "gbdt" or reg_alpha != 0.0 or min_split_gain != 0.0:
        boost = dr_gbdt_boost(DR_GBDT_BOOST[boosting], 0, 0, 0, float(reg_alpha), float(min_split_gain), None, None)
        if boosting == "goss":
            boost.goss_warmup, boost.goss_top_k, boost.goss_other_k = int(1.0 / learning_rate), top_k, other_k
            qscale = qscale / float(1 << goss_shift)
        if boosting == "dart":
            drop_off, drop_iter = dart_schedule(n_iter, learning_rate, seed, drop_rate, max_drop, skip_drop)
            boost.drop_off, boost.drop_iter = drop_off.ctypes.data, drop_iter.ctypes.data
    prm = dr_gbdt_params(n, F, n_classes, n_iter, max_depth, num_leaves, min_data_in_leaf, learning_rate,
                         min_sum_hessian, qscale, float(reg_lambda), float(colsample_bytree), float(subsample),
                         int(subsample_freq), int(seed))
    d_bins = torch.from_numpy(np.ascontiguousarray(bins)).to(device)
    d_yc = torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).to(device) if n_classes >= 2 else None
    d_yv = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float64)).to(device) if n_classes == 1 else None
    d_w = torch.from_numpy(np.ascontiguousarray(weight, dtype=np.float64)).to(device)
    out_nodes = torch.zeros(n_iter * S * MAX_NODES * NODE_DTYPE.itemsize, dtype=torch.uint8, device=device)
    out_counts = torch.zeros(n_iter * S, dtype=torch.int32, device=device)
    if boost is None:
        ws = torch.empty(ctx.gbdt_workspace_bytes(n, S), dtype=torch.uint8, device=device)
        ctx.gbdt_train(prm, d_bins, n_bins, d_yc, d_yv, d_w, init, ws, out_nodes, out_counts)
    else:
        n_drops = int(drop_off[-1]) if boosting == "dart" else 0
        ws = torch.empty(ctx.gbdt_train_ex_workspace_bytes(n, S, n_drops), dtype=torch.uint8, device=device)
        ctx.gbdt_train_ex(prm, boost, d_bins, n_bins, d_yc, d_yv, d_w, init, ws, out_nodes, out_counts)
    nodes = out_nodes.cpu().numpy().view(NODE_DTYPE).reshape(n_iter, S, MAX_NODES)
    counts = out_counts.cpu().numpy().reshape(n_iter, S)
    forest = flatten(nodes, counts, init, bin_values, F, n_classes)
    if k:                                    # back to the target's own units (exact)
        forest["baseline"] = np.ldexp(forest["baseline"], k)
        forest["value"] = np.ldexp(forest["value"], k)
    return forest


def flatten(nodes, counts, init, bin_values, n_features, n_classes):
    """device node records -> flat forest; threshold = midpoint between the split bin's value and the
    next one in the feature's encoded value space."""
    n_iter, S, _ = nodes.shape
    sizes = counts.reshape(-1).astype(np.int64)
    tree_offset = np.zeros(len(sizes) + 1, dtype=np.int64)
    tree_offset[1:] = np.cumsum(sizes)
    keep = (np.arange(MAX_NODES)[None, :] < sizes[:, None]).reshape(-1)
    flat = nodes.reshape(-1)[keep]
    feat = flat["feature"].astype(np.int32)
    leaf = feat < 0
    thr = np.zeros(len(flat))
    # a bin holds one encoded value (1-D entry) or a run of adjacent values (2 x n entry: largest / smallest
    # value of every bin): the threshold sits midway between the split bin's largest and the next bin's smallest
    hi_lo = [(v, v) if np.ndim(v) == 1 else (v[0], v[1]) for v in bin_values]
    max_bins = max(len(h) for h, _ in hi_lo)
    tab_hi, tab_lo = np.zeros((n_features, max_bins + 1)), np.zeros((n_features, max_bins + 1))
    for f, (h, l) in enumerate(hi_lo):
        tab_hi[f, :len(h)] = h
        tab_lo[f, :len(l)] = l
    fi, ti = np.where(leaf, 0, feat), flat["thr_bin"].astype(np.int64)
    hi, lo = tab_hi[fi, ti], tab_lo[fi, np.minimum(ti + 1, max_bins)]
    with np.errstate(invalid="ignore", over="ignore"):
        mid = (hi + lo) / 2.0
    # +-inf neighbours, an overflowing sum or adjacent doubles (continuous features only): the split bin's
    # largest value separates the two sides exactly as well
    thr = np.where(leaf, 0.0, np.where(np.isfinite(mid) & (mid < lo), mid, hi))
    return {
        "n_features": int(n_features), "n_classes": int(n_classes), "baseline": np.asarray(init, dtype=np.float64),
        "tree_seq": np.tile(np.arange(S, dtype=np.int32), n_iter), "tree_offset": tree_offset,
        "feature": feat, "threshold": thr, "missing_left": np.where(leaf, 0, flat["missing_left"]).astype(np.uint8),
        "left": np.where(leaf, 0, flat["left"]).astype(np.int32),
        "right": np.where(leaf, 0, flat["right"]).astype(np.int32),
        "value": np.where(leaf, flat["value"], 0.0).astype(np.float64),
    }
