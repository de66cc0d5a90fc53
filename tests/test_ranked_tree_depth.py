"""Rank-coded forests whose trees differ in depth.  k_forest_predict_ranked walks every tree to the
forest-wide max_depth (a tree that ends earlier stays on its leaf); the forests here mix single-leaf,
shallow and deep trees inside one group of 8 / 16 trees (one deep tree among shallow ones, a group of
single leaves), with sequences whose tree count is not a multiple of 8 or 16, so that any change of
how far each tree is walked is checked against the oracle's tree-order float64 sums."""
import numpy as np
import pytest

import parity_utils  # noqa: F401  (sys.path)

# depth caps of the first 16 boosting rounds: a depth-7 tree among single leaves and stumps, then a
# group of single-leaf trees; later rounds draw 0..7
HEAD = [0, 1, 0, 2, 0, 0, 7, 1, 0, 0, 0, 0, 0, 0, 0, 0]


def depth_caps(rng, n_classes, n_iter):
    S = 1 if n_classes <= 2 else n_classes
    caps = rng.integers(0, 8, size=(n_iter, S))
    caps[:len(HEAD)] = np.asarray(HEAD)[:n_iter, None]
    return caps.ravel()


def mixed_case(rng, doms, n_classes, n_iter, n_rows):
    from repair.forest import encoder_width
    from tools.randforest import mixed_depth_forest
    names = ["a%d" % i for i in range(len(doms))]
    codes = {nm: rng.integers(-1, d, size=n_rows).astype(np.int32) for nm, d in zip(names, doms)}
    encoders = [{"attr": names[i], "type": "sum" if doms[i] < 12 else "ordinal",
                 "categories": [int(c) for c in rng.permutation(doms[i])[:doms[i] - (i % 3 == 0)]]}
                for i in range(1, len(doms))]
    thr = []
    for e in encoders:
        kk = len(e["categories"])
        thr += [[-0.5, 0.5]] * (kk - 1) if e["type"] == "sum" else [[j + 0.5 for j in range(kk)]]
    n_feat = sum(encoder_width(e) for e in encoders)
    forest = mixed_depth_forest(n_feat, n_classes, depth_caps(rng, n_classes, n_iter), thr, rng, leaf_scale=0.1)
    forest["baseline"] = rng.normal(0.0, 0.5, size=len(forest["baseline"]))
    spec = {"forest": forest, "encoders": encoders, "class_codes": list(range(max(n_classes, 2))), "integral": False}
    return names, codes, encoders, forest, spec, dict(zip(names, doms))


# (classes, boosting rounds): one sequence of 45 trees, three of 37, five of 70
CASES = [(2, 45), (3, 37), (5, 70)]


@pytest.mark.parametrize("n_classes,n_iter", CASES)
def test_ranked_image_of_mixed_depth_groups(n_classes, n_iter):
    from oracle.forest import forest_margins
    from ranked_emul import eval_image
    from repair.forest import encode_matrix, group_by_sequence, rank_code, ranked_image
    rng = np.random.default_rng(50 + n_classes)
    names, codes, encoders, forest, spec, dict_sizes = mixed_case(rng, [5, 4, 30, 3, 9, 64, 2], n_classes,
                                                                  n_iter, 200)
    rk = rank_code(spec, dict_sizes)
    off, order = group_by_sequence(forest)
    img = ranked_image(rk, order, off)
    assert set(rk["tree_depth"].tolist()) == set(range(8))
    assert np.all(np.diff(off) % 8 != 0)                           # every sequence ends on a partial group
    hdr = img["tree_hdr"].reshape(-1, 2)
    cto, ch = img["chunk_tree_off"], img["chunk_hdr_off"]
    slot = np.concatenate([ch[c] + np.arange(cto[c + 1] - cto[c]) for c in range(len(cto) - 1)])
    bias = hdr[slot, 1].view(np.int32)
    assert bias.min() < 0 and bias.max() <= 0
    # the value bias in the header is the one the flat image implies
    toff, lo = rk["tree_offset"], rk["tree_leaf_off"]
    sizes, lsizes = (toff[1:] - toff[:-1])[order], (lo[1:] - lo[:-1])[order]
    for c in range(len(cto) - 1):
        a, b = int(cto[c]), int(cto[c + 1])
        node_in = np.r_[0, np.cumsum(sizes[a:b])][:-1]
        leaf_in = np.r_[0, np.cumsum(lsizes[a:b])][:-1]
        assert np.array_equal(bias[a:b], leaf_in - node_in - rk["first_leaf"][order[a:b]])
    got = eval_image(rk, img, forest["baseline"], {nm: codes[nm] for nm in names[1:]})
    want = forest_margins(forest, encode_matrix(encoders, {nm: codes[nm] for nm in names[1:]}, {}, dict_sizes))
    assert np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("n_classes,n_iter", CASES)
def test_ranked_kernel_on_mixed_depth_groups(n_classes, n_iter):
    """All four kernel instantiations, several tiles per CTA."""
    torch = pytest.importorskip("torch")
    from oracle import ckernels
    from repair._native import Context
    from repair.forest import DeviceModel, encode_matrix
    assert ckernels.available(), "oracle/c is not built (run __graft_entry__.build())"
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_rows = sm * 512 * 3 + 4096 + 17
    rng = np.random.default_rng(70 + n_classes)
    names, codes, encoders, forest, spec, dict_sizes = mixed_case(rng, [5, 4, 30, 3, 9, 64, 2], n_classes,
                                                                  n_iter, n_rows)
    tile_np = np.stack([codes[nm] for nm in names], axis=1).astype(np.int32)
    dm = DeviceModel(spec, {nm: i for i, nm in enumerate(names)}, dict_sizes, {}, torch.device("cuda", 0))
    assert dm.ranked is not None
    cells = np.sort(rng.choice(n_rows, size=sm * 512 * 3 + 17, replace=False)).astype(np.int32)
    X = encode_matrix(encoders, {nm: tile_np[cells, i] for i, nm in enumerate(names) if i}, {}, dict_sizes)
    want_m = ckernels.forest_margins(forest, X)
    lab = (want_m[:, 0] > 0).astype(np.int32) if want_m.shape[1] == 1 else np.argmax(want_m, axis=1).astype(np.int32)
    ctx = Context(0)
    try:
        for layout in (0, 1, 2, 3):                                # auto (wide 512 / 8), bytes, wide 8, wide 16
            dm.ranked.layout = layout
            tile = torch.from_numpy(tile_np.copy()).cuda()
            margins = torch.empty((len(cells), dm.n_seq), dtype=torch.float64, device="cuda")
            dm.predict(ctx, tile, len(names), None, 0, torch.from_numpy(cells).cuda(), len(cells), 0, margins)
            assert np.array_equal(margins.cpu().numpy(), want_m), layout
            assert np.array_equal(tile.cpu().numpy()[cells, 0], lab), layout
    finally:
        ctx.close()
