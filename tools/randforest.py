"""Random-init forests of the reference's architecture (TEST / BENCH infrastructure, not product
code): ``n_iter`` boosting rounds x one tree per class, depth <= 7, <= 31 leaves -- the shape
``train.py:102-115`` of the reference fixes.  Used by the kernel parity tests (irregular topologies
stress the forest kernels harder than trained, level-wise trees do) and by ``bench.py --forests
random``."""
import numpy as np


def _random_shape(rng, max_depth, max_leaves):
    """One random tree topology: arrays (left, right, depth) with -1 children on leaves."""
    left, right, depth = [-1], [-1], [0]
    leaves = [0]
    while len(leaves) < max_leaves:
        cand = [n for n in leaves if depth[n] < max_depth]
        if not cand:
            break
        n = cand[int(rng.integers(len(cand)))]
        left[n], right[n] = len(left), len(left) + 1
        for _ in range(2):
            left.append(-1), right.append(-1), depth.append(depth[n] + 1)
        leaves.remove(n)
        leaves += [len(left) - 2, len(left) - 1]
    return np.array(left), np.array(right)


def random_forest(n_features, n_classes, n_iter, feature_thresholds, rng, max_depth=7, max_leaves=31,
                  leaf_scale=0.01, n_shapes=16):
    """Random-init forest of the reference's architecture (n_iter boosting rounds x one tree per
    class, depth <= max_depth, <= max_leaves leaves): used by bench.py where no training data of
    the named size can be fitted in the time budget.  ``feature_thresholds[f]`` lists the split
    points that make sense for encoded feature f.  Trees draw their topology from a pool of
    `n_shapes` random shapes; split features, thresholds, NaN directions and leaf values are
    independent per tree."""
    S = 1 if n_classes <= 2 else n_classes
    T = n_iter * S
    usable = np.array([f for f in range(n_features) if len(feature_thresholds[f])], dtype=np.int64)
    shapes = [_random_shape(rng, max_depth if len(usable) else 0, max_leaves) for _ in range(n_shapes)]
    sizes = np.array([len(sh[0]) for sh in shapes])
    shape_of = rng.integers(0, n_shapes, size=T)
    tree_sizes = sizes[shape_of]
    tree_offset = np.zeros(T + 1, dtype=np.int64)
    tree_offset[1:] = np.cumsum(tree_sizes)
    M = int(tree_offset[-1])
    feature = np.full(M, -1, dtype=np.int32)
    threshold = np.zeros(M)
    missing_left = np.zeros(M, dtype=np.uint8)
    left = np.zeros(M, dtype=np.int32)
    right = np.zeros(M, dtype=np.int32)
    value = np.zeros(M)
    max_thr = max([len(t) for t in feature_thresholds] + [1])
    thr_tab = np.zeros((max(n_features, 1), max_thr))
    thr_len = np.ones(max(n_features, 1), dtype=np.int64)
    for f, t in enumerate(feature_thresholds):
        if len(t):
            thr_tab[f, :len(t)] = t
            thr_len[f] = len(t)
    for si, (l, r) in enumerate(shapes):
        trees = np.nonzero(shape_of == si)[0]
        if len(trees) == 0:
            continue
        idx = tree_offset[trees][:, None] + np.arange(len(l))[None, :]        # [n_trees, nodes]
        internal = l >= 0
        n_int = int(internal.sum())
        left[idx] = np.where(internal, l, 0)[None, :]
        right[idx] = np.where(internal, r, 0)[None, :]
        if n_int:
            f = usable[rng.integers(0, len(usable), size=(len(trees), n_int))]
            u = rng.random(size=f.shape)
            th = thr_tab[f, np.minimum((u * thr_len[f]).astype(np.int64), thr_len[f] - 1)]
            feature[idx[:, internal]] = f
            threshold[idx[:, internal]] = th
            missing_left[idx[:, internal]] = rng.integers(0, 2, size=f.shape)
        value[idx[:, ~internal]] = rng.normal(0.0, leaf_scale, size=(len(trees), int((~internal).sum())))
    return {
        "n_features": int(n_features), "n_classes": int(n_classes), "baseline": np.zeros(S),
        "tree_seq": (np.arange(T) % S).astype(np.int32), "tree_offset": tree_offset,
        "feature": feature, "threshold": threshold, "missing_left": missing_left, "left": left, "right": right,
        "value": value,
    }


def mixed_depth_forest(n_features, n_classes, depth_caps, feature_thresholds, rng, leaf_scale=0.01):
    """Random forest whose tree t (boosting order: round-major, one tree per class) is at most
    ``depth_caps[t]`` deep (<= 31 leaves; a cap of 0 is a single leaf): forests that mix single-leaf,
    shallow and deep trees in any pattern, for the ranked kernel's per-tree walk depth."""
    caps = np.asarray(depth_caps, dtype=np.int64)
    S = 1 if n_classes <= 2 else n_classes
    assert len(caps) % S == 0
    pool = {int(d): random_forest(n_features, 2, int((caps == d).sum()), feature_thresholds, rng, max_depth=int(d),
                                  leaf_scale=leaf_scale)
            for d in np.unique(caps)}
    used = {d: 0 for d in pool}
    keys = ("feature", "threshold", "missing_left", "left", "right", "value")
    parts = {k: [] for k in keys}
    sizes = []
    for d in caps.tolist():
        f = pool[d]
        a, b = int(f["tree_offset"][used[d]]), int(f["tree_offset"][used[d] + 1])
        used[d] += 1
        for k in keys:
            parts[k].append(f[k][a:b])
        sizes.append(b - a)
    tree_offset = np.zeros(len(caps) + 1, dtype=np.int64)
    tree_offset[1:] = np.cumsum(sizes)
    out = {k: np.concatenate(v) for k, v in parts.items()}
    out.update({"n_features": int(n_features), "n_classes": int(n_classes), "baseline": np.zeros(S),
                "tree_seq": (np.arange(len(caps)) % S).astype(np.int32), "tree_offset": tree_offset})
    return out
