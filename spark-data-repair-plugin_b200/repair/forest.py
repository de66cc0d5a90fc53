"""Flat forest exchange format, feature encoders and their device images.

The reference hands its pandas UDF pickled LightGBM models plus ``category_encoders`` transformers
(``model.py:1067-1073,1111-1133``); here a model is a handful of flat arrays the CUDA kernel
walks directly (``dr_forest`` in ``include/b200repair.h``).

Flat forest (host, NumPy):
  n_classes      1 = regression, 2 = binary (one tree sequence), C > 2 = C sequences
  baseline       float64[S]
  tree_seq       int32[T]        sequence (class) of tree t, trees in boosting order
  tree_offset    int64[T+1]      node range of tree t
  feature        int32[M]  (-1 = leaf)   threshold float64[M]   missing_left uint8[M]
  left, right    int32[M]  (relative to the tree root)          value float64[M] (leaf value)
Encoders (one per feature column, in feature order):
  {"attr", "type": "cont"}                          float passthrough, NaN = NULL
  {"attr", "type": "ordinal", "categories": [...]}  first-seen order on the training sample ->
                                                    1..k; NULL never seen -> -2; unseen value -> NaN
  {"attr", "type": "sum", "categories": [...]}      deviation (sum) contrast, k-1 columns, last
                                                    level = -1 row; NULL never seen -> zeros; unseen -> NaN
  categories hold dictionary CODES (-1 = the NULL category).
"""
import os

import numpy as np

LEAF = 0xFFF
MAX_TREE_NODES = 511


def first_seen(codes):
    """Distinct values of a code array in order of first appearance (pandas ``unique`` order)."""
    codes = np.asarray(codes)
    _, idx = np.unique(codes, return_index=True)
    return [int(c) for c in codes[np.sort(idx)]]


def encoder_type(attr, continuous, domain_stats, small_domain_threshold):
    # model.py:701-729: SumEncoder for ndv < small_domain_threshold, OrdinalEncoder otherwise
    if attr in continuous:
        return "cont"
    return "sum" if int(domain_stats[attr]) < small_domain_threshold else "ordinal"


def encoder_width(enc):
    if enc["type"] == "sum":
        k = len(enc["categories"])
        return k - 1 if k >= 2 else 0
    return 1


def encoder_lut(enc, dict_size):
    """float64 [dict_size + 1, width]: row (code + 1) = encoded feature values of that code."""
    w = encoder_width(enc)
    lut = np.full((dict_size + 1, w), np.nan, dtype=np.float64)
    cats = enc["categories"]
    null_seen = -1 in cats
    if enc["type"] == "ordinal":
        for pos, c in enumerate(cats):
            lut[c + 1, 0] = float(pos + 1)
        if not null_seen:
            lut[0, 0] = -2.0
        return lut
    k = len(cats)
    if k < 2:
        return lut
    for pos, c in enumerate(cats):
        row = np.zeros(k - 1)
        if pos == k - 1:
            row[:] = -1.0
        else:
            row[pos] = 1.0
        lut[c + 1] = row
    if not null_seen:
        lut[0] = 0.0
    return lut


def encode_matrix(encoders, code_cols, value_cols, dict_sizes):
    """Host-side encoding of a sample: code_cols / value_cols are {attr: array}.  -> float64 [n, F']"""
    n = 0
    for e in encoders:
        src = value_cols if e["type"] == "cont" else code_cols
        n = len(src[e["attr"]])
        break
    blocks = []
    for e in encoders:
        if e["type"] == "cont":
            blocks.append(np.asarray(value_cols[e["attr"]], dtype=np.float64).reshape(-1, 1))
        else:
            lut = encoder_lut(e, dict_sizes[e["attr"]])
            blocks.append(lut[np.asarray(code_cols[e["attr"]], dtype=np.int64) + 1])
    if not blocks:
        return np.zeros((n, 0))
    return np.concatenate(blocks, axis=1)


def pack_nodes(forest):
    """-> (node_thr float64[M], node_meta uint32[M]) in the kernel's packed layout."""
    feat = np.asarray(forest["feature"], dtype=np.int64)
    if feat.size and feat.max() >= LEAF:
        raise ValueError("too many encoded features for the packed node format")
    left = np.asarray(forest["left"], dtype=np.int64)
    right = np.asarray(forest["right"], dtype=np.int64)
    if left.size and (left.max() > MAX_TREE_NODES or right.max() > MAX_TREE_NODES):
        raise ValueError("a tree has more than {} nodes".format(MAX_TREE_NODES))
    is_leaf = feat < 0
    meta = np.where(is_leaf, LEAF, feat).astype(np.uint32)
    meta |= (np.asarray(forest["missing_left"], dtype=np.uint32) & 1) << 12
    meta |= (np.where(is_leaf, 0, left).astype(np.uint32) & 0x1FF) << 13
    meta |= (np.where(is_leaf, 0, right).astype(np.uint32) & 0x1FF) << 22
    thr = np.where(is_leaf, forest["value"], forest["threshold"]).astype(np.float64)
    return thr, meta


def group_by_sequence(forest):
    """Reorders trees so that each sequence is contiguous (boosting order kept inside a sequence).
    -> (seq_tree_off int32[S+1], tree order int array)"""
    seq = np.asarray(forest["tree_seq"], dtype=np.int64)
    S = len(forest["baseline"])
    order = np.argsort(seq, kind="stable")
    counts = np.bincount(seq, minlength=S)
    off = np.zeros(S + 1, dtype=np.int32)
    off[1:] = np.cumsum(counts)
    return off, order


def bfs_relabel(toff, left, right, is_leaf):
    """Breadth-first renumbering of every tree at once: root = 0 and the right child of a node is its
    left child + 1 (what the carry-coded node word needs).  -> (new tree-relative index per node, -1
    for nodes the root does not reach; nodes kept per tree; depth of every tree = its deepest leaf)."""
    toff = np.asarray(toff, dtype=np.int64)
    n_trees = len(toff) - 1
    new = np.full(len(left), -1, dtype=np.int64)
    kept = np.ones(n_trees, dtype=np.int64)
    tree_depth = np.zeros(n_trees, dtype=np.int64)
    if n_trees == 0:
        return new, kept, tree_depth
    frontier, ftree = toff[:-1].copy(), np.arange(n_trees, dtype=np.int64)
    new[frontier] = 0
    depth = 0
    while True:
        inner = ~is_leaf[frontier]
        if not inner.any():
            break
        fr, tr = frontier[inner], ftree[inner]                 # grouped by tree, level order inside a tree
        start = np.flatnonzero(np.r_[True, tr[1:] != tr[:-1]])
        cnt = np.diff(np.r_[start, len(tr)])
        k = np.arange(len(tr)) - np.repeat(start, cnt)
        base = kept[tr] + 2 * k
        lch, rch = toff[tr] + left[fr], toff[tr] + right[fr]
        new[lch], new[rch] = base, base + 1
        kept[tr[start]] += 2 * cnt
        frontier, ftree = np.stack([lch, rch], axis=1).ravel(), np.repeat(tr, 2)
        depth += 1
        tree_depth[tr[start]] = depth
    return new, kept, tree_depth


def forest_shape_stats(forest):
    """Shape of a flat forest (host, for bench.py / DESIGN.md): how much of a fixed-depth walk is
    needed.  -> dict(n_trees, max_depth, mean_tree_depth, single_leaf_tree_frac, mean_leaves,
    mean_leaf_depth = unweighted mean depth of the leaves)."""
    toff = np.asarray(forest["tree_offset"], dtype=np.int64)
    feat = np.asarray(forest["feature"], dtype=np.int64)
    left, right = np.asarray(forest["left"], dtype=np.int64), np.asarray(forest["right"], dtype=np.int64)
    n_trees = len(toff) - 1
    if n_trees == 0:
        return {"n_trees": 0, "max_depth": 0, "mean_tree_depth": 0.0, "single_leaf_tree_frac": 0.0,
                "mean_leaves": 0.0, "mean_leaf_depth": 0.0}
    is_leaf = feat < 0
    _, _, tree_depth = bfs_relabel(toff, left, right, is_leaf)
    node_depth = np.full(len(feat), -1, dtype=np.int64)
    frontier = toff[:-1].copy()
    sizes = toff[1:] - toff[:-1]
    tree_of = np.repeat(np.arange(n_trees), sizes)
    node_depth[frontier] = 0
    d = 0
    while len(frontier):
        inner = frontier[~is_leaf[frontier]]
        if not len(inner):
            break
        base = toff[tree_of[inner]]
        frontier = np.concatenate([base + left[inner], base + right[inner]])
        d += 1
        node_depth[frontier] = d
    reach = is_leaf & (node_depth >= 0)
    leaves_per_tree = np.bincount(tree_of[reach], minlength=n_trees)
    return {"n_trees": int(n_trees), "max_depth": int(tree_depth.max()),
            "mean_tree_depth": float(tree_depth.mean()),
            "single_leaf_tree_frac": float((leaves_per_tree <= 1).mean()),
            "mean_leaves": float(leaves_per_tree.mean()),
            "mean_leaf_depth": float(node_depth[reach].mean())}


def pair_order(kept, is_leaf_new_order):
    """Final tree-relative node order for the rank-coded image: the root, then the sibling pairs
    (breadth-first numbering of bfs_relabel: pair p of a tree = nodes 2p+1, 2p+2) stably sorted by class --
    two internal nodes, one of each, two leaves -- so that every leaf of a tree sits in the tail
    [first_leaf, n_nodes) and the leaf-value array indexed by `node - first_leaf` wastes at most one
    slot per mixed pair.  kept: nodes per tree; is_leaf_new_order: leaf flag per node in breadth-first
    order (all trees concatenated).  -> (final index per node in that order, first_leaf per tree)."""
    n_trees = len(kept)
    starts = np.zeros(n_trees + 1, dtype=np.int64)
    starts[1:] = np.cumsum(kept)
    n_pairs = (kept - 1) // 2
    pstart = np.zeros(n_trees + 1, dtype=np.int64)
    pstart[1:] = np.cumsum(n_pairs)
    ptree = np.repeat(np.arange(n_trees), n_pairs)
    pidx = np.arange(int(pstart[-1])) - pstart[ptree]                 # pair number inside its tree
    lpos = starts[ptree] + 1 + 2 * pidx                               # left node of the pair (new order)
    pclass = is_leaf_new_order[lpos].astype(np.int64) + is_leaf_new_order[lpos + 1].astype(np.int64)
    order = np.lexsort((pidx, pclass, ptree))                          # stable inside (tree, class)
    rank_in_tree = np.empty(len(order), dtype=np.int64)
    rank_in_tree[order] = np.arange(len(order)) - pstart[ptree[order]]
    fin = np.zeros(int(starts[-1]), dtype=np.int64)                    # roots stay at 0
    fin[lpos] = 1 + 2 * rank_in_tree
    fin[lpos + 1] = 2 + 2 * rank_in_tree
    tree_of = np.repeat(np.arange(n_trees), kept)
    big = np.iinfo(np.int64).max
    first_leaf = np.full(n_trees, big, dtype=np.int64)
    np.minimum.at(first_leaf, tree_of[is_leaf_new_order], fin[is_leaf_new_order])
    return fin, first_leaf


def rank_code(spec, dict_sizes):
    """Rank-coded image of an all-discrete model for dr_forest_predict_ranked, or None when the
    model does not qualify (continuous feature, > 253 distinct values per feature, > 255 rank slots).
    Decisions are unchanged: `x <= thr` <=> `rank(x) < #values <= thr`.

    A rank SLOT is one (encoded feature, NaN direction) combination that some node of the forest
    actually tests: its LUT maps a dictionary code (+1) to rank + 1 (1..254), with NaN already folded
    to 0 (nodes that send NaN left) or 255 (right).  Features no node tests get no slot.
    Nodes of a tree are ordered by pair_order(); `word` holds the node words with TREE-relative child
    indices (ranked_image rebases them to the chunk):
      internal  slot << 24 | left child << 8 | (256 - (thr_rank + 1))     right child = left child + 1
      leaf      own index << 8                                            (slot 0, never carries)
    so that `word + rank` carries into the child field exactly when the row goes right, and a leaf
    stays where it is.  `leaf_value` holds, per tree, the values of nodes first_leaf .. n_nodes-1
    (0 for the few internal nodes in that range): the value of the node a walk ends on is
    leaf_value[tree_leaf_off[t] + node - first_leaf[t]], no look-up of the leaf's own word needed."""
    f = spec["forest"]
    encoders = spec["encoders"]
    if any(e["type"] == "cont" for e in encoders) or spec.get("class_codes") is None:
        return None
    luts, feat_attr = [], []
    for e in encoders:
        lut = encoder_lut(e, dict_sizes[e["attr"]])
        for j in range(lut.shape[1]):
            luts.append(lut[:, j])
            feat_attr.append(e["attr"])
    n_feat = len(luts)
    if n_feat != int(f["n_features"]):
        return None
    toff = np.asarray(f["tree_offset"], dtype=np.int64)
    feat = np.asarray(f["feature"], dtype=np.int64)
    is_leaf = feat < 0
    left, right = np.asarray(f["left"], dtype=np.int64), np.asarray(f["right"], dtype=np.int64)
    ml_all = np.asarray(f["missing_left"], dtype=np.int64) & 1
    new, kept, tree_depth = bfs_relabel(toff, left, right, is_leaf)
    depth = int(tree_depth.max()) if len(tree_depth) else 0
    new_toff = np.zeros(len(toff), dtype=np.int64)
    new_toff[1:] = np.cumsum(kept)
    old_sizes = toff[1:] - toff[:-1]
    tree_of = np.repeat(np.arange(len(old_sizes)), old_sizes)
    live = new >= 0
    pos = new_toff[tree_of[live]] + new[live]                      # BFS slot of every kept node
    src_bfs = np.empty(int(new_toff[-1]), dtype=np.int64)
    src_bfs[pos] = np.flatnonzero(live)                            # old node stored in each BFS slot
    fin_bfs, first_leaf = pair_order(kept, is_leaf[src_bfs])
    n_tree_bfs = tree_of[src_bfs]
    src = np.empty_like(src_bfs)
    src[new_toff[n_tree_bfs] + fin_bfs] = src_bfs                  # old node stored in each FINAL slot
    fin_of_old = np.full(len(feat), -1, dtype=np.int64)
    fin_of_old[src_bfs] = fin_bfs
    # rank slots: the (feature, NaN direction) combinations the reachable internal nodes test
    used = live & ~is_leaf
    combo = np.unique(feat[used] * 2 + ml_all[used])
    if len(combo) > 255:
        return None
    slot_of = np.full(2 * max(n_feat, 1), 0, dtype=np.int64)
    slot_of[combo] = np.arange(len(combo))
    rank_lut, rank_off, slot_attr, slot_nan, values = [], [0], [], [], {}
    for cb in combo.tolist():
        j, nan_left = cb >> 1, cb & 1
        col = luts[j]
        if j not in values:
            values[j] = np.unique(col[~np.isnan(col)])
        vals = values[j]
        if len(vals) > 253:
            return None
        nan_byte = 0 if nan_left else 255
        r = np.full(len(col), nan_byte, dtype=np.uint8)
        ok = ~np.isnan(col)
        r[ok] = (np.searchsorted(vals, col[ok]) + 1).astype(np.uint8)  # ranks are stored +1 (1..254)
        rank_lut.append(r)
        rank_off.append(rank_off[-1] + len(r))
        slot_attr.append(feat_attr[j])
        slot_nan.append(nan_byte)
    thr = np.asarray(f["threshold"], dtype=np.float64)
    thr_rank = np.zeros(len(feat), dtype=np.int64)
    for j in values:  # number of distinct values <= threshold, per feature
        m = used & (feat == j)
        thr_rank[m] = np.searchsorted(values[j], thr[m], side="right")
    n_leaf = is_leaf[src]
    n_tree = tree_of[src]
    own = np.arange(len(src), dtype=np.int64) - new_toff[n_tree]
    child = fin_of_old[np.where(n_leaf, src, toff[n_tree] + left[src])]   # left child, tree relative
    cthr = 256 - (thr_rank[src] + 1)                               # thr in 1..254 -> 2..255
    slot = slot_of[np.where(n_leaf, 0, feat[src] * 2 + ml_all[src])]
    internal = (slot << 24) | (child << 8) | cthr
    leaf = own << 8
    word = np.where(n_leaf, leaf, internal).astype(np.uint32)
    n_vals = kept - first_leaf                                     # value slots per tree
    tree_leaf_off = np.zeros(len(toff), dtype=np.int64)
    tree_leaf_off[1:] = np.cumsum(n_vals)
    leaf_value = np.zeros(int(tree_leaf_off[-1]), dtype=np.float64)
    vpos = tree_leaf_off[n_tree] + own - first_leaf[n_tree]
    leaf_value[vpos[n_leaf]] = np.asarray(f["value"], dtype=np.float64)[src][n_leaf]
    return {"word": word, "tree_offset": new_toff, "leaf_value": leaf_value, "tree_leaf_off": tree_leaf_off,
            "first_leaf": first_leaf, "rank_lut": np.concatenate(rank_lut) if rank_lut else np.zeros(1, np.uint8),
            "rank_lut_off": np.asarray(rank_off, dtype=np.int32), "slot_attr": slot_attr,
            "slot_nan": np.asarray(slot_nan if slot_nan else [0], dtype=np.uint8), "n_slots": len(combo),
            "max_depth": depth, "tree_depth": tree_depth}


# DR_RANKED_CHUNK_* in include/b200repair.h
RANKED_CHUNK_NODES, RANKED_CHUNK_LEAVES, RANKED_CHUNK_TREES, RANKED_GROUP = 4096, 2560, 256, 16


def ranked_image(rk, order, seq_tree_off):
    """Device layout of a rank-coded forest: trees grouped by sequence (`order`) and cut into chunks
    of whole trees that fit the kernel's shared-memory buffers (never straddling a sequence; a
    multiple of RANKED_GROUP trees except at the end of a sequence).  Every chunk starts on a 16-byte
    boundary of the node / leaf-plane / header arrays (TMA granules); child indices are rebased to the
    chunk; tree_hdr holds, per tree, (root word, value bias) relative to the chunk: the value of the
    chunk-relative node c a walk ends on is leaf[chunk_leaf_off + bias + c] (bias is a signed int32)."""
    toff = np.asarray(rk["tree_offset"], dtype=np.int64)
    lo = np.asarray(rk["tree_leaf_off"], dtype=np.int64)
    order = np.asarray(order, dtype=np.int64)
    n_sizes = (toff[1:] - toff[:-1])[order]
    l_sizes = (lo[1:] - lo[:-1])[order]
    nc, lc = np.r_[0, np.cumsum(n_sizes)], np.r_[0, np.cumsum(l_sizes)]
    chunk_tree_off, chunk_seq = [0], []
    for s in range(len(seq_tree_off) - 1):
        t, t_end = int(seq_tree_off[s]), int(seq_tree_off[s + 1])
        while t < t_end:
            hi_n = int(np.searchsorted(nc, nc[t] + RANKED_CHUNK_NODES, side="right")) - 1
            hi_l = int(np.searchsorted(lc, lc[t] + RANKED_CHUNK_LEAVES, side="right")) - 1
            hi = min(hi_n, hi_l, t + RANKED_CHUNK_TREES)
            if hi < t_end:
                hi = t + max((hi - t) // RANKED_GROUP * RANKED_GROUP, 1)
            hi = max(t + 1, min(hi, t_end))
            if nc[hi] - nc[t] > RANKED_CHUNK_NODES or lc[hi] - lc[t] > RANKED_CHUNK_LEAVES:
                raise ValueError("a tree does not fit the ranked kernel's chunk buffers")
            chunk_tree_off.append(hi)
            chunk_seq.append(s)
            t = hi
    cto = np.asarray(chunk_tree_off, dtype=np.int64)
    c_nodes, c_leaves, c_trees = nc[cto[1:]] - nc[cto[:-1]], lc[cto[1:]] - lc[cto[:-1]], cto[1:] - cto[:-1]
    chunk_node_off = np.r_[0, np.cumsum((c_nodes + 3) // 4 * 4)]
    chunk_leaf_off = np.r_[0, np.cumsum((c_leaves + 3) // 4 * 4)]
    chunk_hdr_off = np.r_[0, np.cumsum((c_trees + 1) // 2 * 2)]
    chunk_of_tree = np.repeat(np.arange(len(c_trees)), c_trees)
    node_in_chunk = nc[:-1] - nc[cto[:-1]][chunk_of_tree]          # first node of each tree, chunk relative
    leaf_in_chunk = lc[:-1] - lc[cto[:-1]][chunk_of_tree]
    word = np.zeros(max(int(chunk_node_off[-1]), 4), dtype=np.uint32)
    leaf = np.zeros(max(int(chunk_leaf_off[-1]), 4), dtype=np.float64)
    hdr = np.zeros((max(int(chunk_hdr_off[-1]), 2), 2), dtype=np.uint32)
    tree_new = np.repeat(np.arange(len(order)), n_sizes)
    within = np.arange(int(n_sizes.sum())) - np.repeat(nc[:-1], n_sizes)
    src = np.repeat(toff[:-1][order], n_sizes) + within
    rebased = rk["word"][src].astype(np.int64) + (node_in_chunk[tree_new] << 8)
    word[chunk_node_off[chunk_of_tree[tree_new]] + node_in_chunk[tree_new] + within] = rebased.astype(np.uint32)
    ltree_new = np.repeat(np.arange(len(order)), l_sizes)
    lwithin = np.arange(int(l_sizes.sum())) - np.repeat(lc[:-1], l_sizes)
    lsrc = np.repeat(lo[:-1][order], l_sizes) + lwithin
    leaf[chunk_leaf_off[chunk_of_tree[ltree_new]] + leaf_in_chunk[ltree_new] + lwithin] = rk["leaf_value"][lsrc]
    slot = chunk_hdr_off[chunk_of_tree] + (np.arange(len(order)) - cto[:-1][chunk_of_tree])
    roots = chunk_node_off[chunk_of_tree] + node_in_chunk
    hdr[slot, 0] = word[roots] if len(order) else 0
    bias = leaf_in_chunk - (node_in_chunk + np.asarray(rk["first_leaf"], dtype=np.int64)[order])
    hdr[slot, 1] = bias.astype(np.int32).view(np.uint32) if len(order) else 0
    # device form of the leaf table: per chunk the low words of its float64 values, then the high words
    # (two 32-bit planes: conflict-free shared-memory loads, see forest_ranked.cu)
    halves = leaf.view(np.uint32).reshape(-1, 2)
    split = np.zeros(2 * len(leaf), dtype=np.uint32)
    for c in range(len(c_trees)):
        a, b = int(chunk_leaf_off[c]), int(chunk_leaf_off[c + 1])
        split[2 * a:2 * a + (b - a)] = halves[a:b, 0]
        split[2 * a + (b - a):2 * b] = halves[a:b, 1]
    return {"word": word, "leaf": leaf, "leaf_split": split, "tree_hdr": hdr.reshape(-1),
            "chunk_tree_off": cto.astype(np.int32), "chunk_seq": np.asarray(chunk_seq, dtype=np.int32),
            "chunk_node_off": chunk_node_off.astype(np.int32), "chunk_leaf_off": chunk_leaf_off.astype(np.int32),
            "chunk_hdr_off": chunk_hdr_off.astype(np.int32)}


class DeviceModel:
    """Device image of one repair model (forest + encoder LUTs) ready for dr_forest_predict."""

    def __init__(self, spec, feature_tile_cols, dict_sizes, cont_tile_cols, device):
        """spec: {"forest", "encoders", "class_codes" or None, "integral"}.
        feature_tile_cols: {attr: column index in the code tile};  cont_tile_cols: {attr: index in
        the float64 tile}."""
        import torch
        from ._native import dr_forest
        f = spec["forest"]
        off, order = group_by_sequence(f)
        thr, meta = pack_nodes(f)
        toff = np.asarray(f["tree_offset"], dtype=np.int64)
        sizes = (toff[1:] - toff[:-1])[order]
        new_off = np.zeros(len(order) + 1, dtype=np.int64)
        new_off[1:] = np.cumsum(sizes)
        idx = np.concatenate([np.arange(toff[t], toff[t + 1]) for t in order]) if len(order) else \
            np.zeros(0, dtype=np.int64)
        thr, meta = thr[idx], meta[idx]
        feat_col, lut_off, luts = [], [0], []
        for e in spec["encoders"]:
            w = encoder_width(e)
            if e["type"] == "cont":
                feat_col.append(-cont_tile_cols[e["attr"]] - 1)
                lut_off.append(lut_off[-1])
                continue
            lut = encoder_lut(e, dict_sizes[e["attr"]])
            for j in range(w):
                feat_col.append(feature_tile_cols[e["attr"]])
                luts.append(lut[:, j])
                lut_off.append(lut_off[-1] + lut.shape[0])
        n_feat = len(feat_col)
        # largest float64-tile column a walk reads (-1: none); predict() checks the tile it is given covers it
        self.max_ccol = max([-c - 1 for c in feat_col if c < 0], default=-1)
        if n_feat != int(f["n_features"]):
            raise ValueError("encoder layout ({} features) does not match the forest ({})".format(
                n_feat, int(f["n_features"])))

        def dev(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)

        self._keep = {
            "seq_tree_off": dev(off, np.int32),
            "tree_node_off": dev(new_off, np.int32),
            "node_thr": dev(thr if len(thr) else np.zeros(1), np.float64),
            "node_meta": dev((meta if len(meta) else np.zeros(1, dtype=np.uint32)).view(np.int32), np.int32),
            "baseline": dev(f["baseline"], np.float64),
            "feat_col": dev(feat_col if feat_col else [0], np.int32),
            "enc_lut_off": dev(lut_off, np.int32),
            "enc_lut": dev(np.concatenate(luts) if luts else np.zeros(1), np.float64),
        }
        cc = spec.get("class_codes")
        self.kind = 0 if cc is not None else 1
        self._keep["class_code"] = dev(cc if cc is not None else [0], np.int32)
        s = dr_forest()
        s.n_seq, s.n_trees, s.n_nodes, s.n_feat = len(f["baseline"]), len(order), len(thr), n_feat
        for k in ("seq_tree_off", "tree_node_off", "node_thr", "node_meta", "baseline", "feat_col", "enc_lut_off",
                  "enc_lut", "class_code"):
            setattr(s, k, self._keep[k].data_ptr())
        s.kind = self.kind
        s.integral = 1 if spec.get("integral") else 0
        s.n_classes = len(cc) if cc is not None else 0
        self.struct = s
        self.n_seq = s.n_seq
        self.n_trees = s.n_trees
        self.n_nodes = s.n_nodes
        self.ranked = None
        rk = rank_code(spec, dict_sizes) if self.kind == 0 else None
        img = None
        if rk is not None and len(order) and np.all(np.diff(off) > 0):
            try:
                img = ranked_image(rk, order, off)
            except ValueError:  # a tree larger than a chunk buffer: the generic kernel takes the model
                img = None
        if img is not None:
            from ._native import dr_forest_ranked
            self._keep.update({
                "r_node_word": dev(img["word"].view(np.int32), np.int32),
                "r_leaf_value": dev(img["leaf_split"].view(np.int32), np.int32),
                "r_chunk_tree_off": dev(img["chunk_tree_off"], np.int32),
                "r_chunk_seq": dev(img["chunk_seq"], np.int32),
                "r_chunk_node_off": dev(img["chunk_node_off"], np.int32),
                "r_chunk_leaf_off": dev(img["chunk_leaf_off"], np.int32),
                "r_chunk_hdr_off": dev(img["chunk_hdr_off"], np.int32),
                "r_tree_hdr": dev(img["tree_hdr"].view(np.int32), np.int32),
                "r_rank_lut": dev(rk["rank_lut"], np.uint8),
                "r_rank_lut_off": dev(rk["rank_lut_off"], np.int32),
                "r_slot_col": dev([feature_tile_cols[a] for a in rk["slot_attr"]] or [0], np.int32),
                "r_slot_nan": dev(rk["slot_nan"], np.uint8),
            })
            r = dr_forest_ranked()
            r.n_seq, r.n_trees, r.n_nodes, r.n_leaves = s.n_seq, s.n_trees, len(img["word"]), len(img["leaf"])
            r.n_slots, r.max_depth, r.n_chunks = int(rk["n_slots"]), int(rk["max_depth"]), len(img["chunk_seq"])
            # DR_RANKED_LAYOUT=bytes|wide8|wide16 pins the shared-memory rank tile (profiling aid)
            r.layout = {"": 0, "bytes": 1, "wide8": 2, "wide16": 3}[os.environ.get("DR_RANKED_LAYOUT", "")]
            for field, key in (("chunk_tree_off", "r_chunk_tree_off"), ("chunk_seq", "r_chunk_seq"),
                               ("chunk_node_off", "r_chunk_node_off"), ("chunk_leaf_off", "r_chunk_leaf_off"),
                               ("chunk_hdr_off", "r_chunk_hdr_off"), ("tree_hdr", "r_tree_hdr"),
                               ("node_word", "r_node_word"), ("leaf_value", "r_leaf_value"),
                               ("baseline", "baseline"), ("slot_col", "r_slot_col"),
                               ("rank_lut_off", "r_rank_lut_off"), ("rank_lut", "r_rank_lut"),
                               ("slot_nan", "r_slot_nan"),
                               ("class_code", "class_code")):
                setattr(r, field, self._keep[key].data_ptr())
            r.n_classes = s.n_classes
            self.ranked = r

    def predict(self, ctx, tile, n_cols, ctile, n_ccols, cells, n_cells, target_col, out_margin=None,
                force_generic=False):
        """Fills the target column of the listed tile rows in place (rank-coded kernel when the model
        qualifies, the generic float64 kernel otherwise).  A model with a continuous feature or target needs
        the float64 tile (ctile, n_ccols columns): the kernel reads it without a check of its own."""
        if self.max_ccol >= 0 and (ctile is None or n_ccols <= self.max_ccol):
            raise ValueError("the model reads float64 tile column {} but got {}".format(
                self.max_ccol, "no float64 tile" if ctile is None else "{} columns".format(n_ccols)))
        if self.kind == 1 and ctile is None:
            raise ValueError("a regressor writes its predictions to the float64 tile, but got none")
        if self.ranked is not None and not force_generic:
            ctx.forest_predict_ranked(self.ranked, tile, n_cols, cells, n_cells, target_col, out_margin)
        else:
            ctx.forest_predict(self.struct, tile, n_cols, ctile, n_ccols, cells, n_cells, target_col, out_margin)
