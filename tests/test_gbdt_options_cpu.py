"""The GPU trainer's boosting options (model.lgb.boosting_type, reg_alpha, min_split_gain, max_bin) in their
specification oracle/gbdt_boost.py and in the host code of repair/gbdt.py.  No GPU needed."""
import hashlib
import logging

import numpy as np
import pytest

from oracle import gbdt as OG
from oracle import gbdt_boost as OB

# sha256 of oracle/gbdt.py's flat forests on problem(3, 1500) / problem(1, 1200) before the options existed
PARENT_SHA = {3: "9fee6cd41ca59ebc2448f203c8139a2ea0915865ddd0b490b4b4213c8d458b2a",
              1: "8df1f30994720e20382bf7680667febda90e641bcafe2d2af66ea03237ca410d"}
DOMS = [4, 9, 3, 6, 30, 2, 12]


def problem(n_classes, n, seed=None):
    """-> (bins, n_bins, bin values, y, class weights or None): the seeded problems of the trainer's
    bit-for-bit tests (tests/test_gpu_kernels.py)."""
    rng = np.random.default_rng(n_classes * 31 + n if seed is None else seed)
    vals = [np.sort(rng.choice(np.arange(-3, 40), size=d, replace=False)).astype(np.float64) for d in DOMS]
    n_bins = np.array([d + 1 for d in DOMS], dtype=np.int32)
    bins = np.stack([rng.integers(0, d + 1, size=n) for d in DOMS], axis=1).astype(np.uint8)
    sig = (bins[:, 0].astype(int) * 3 + bins[:, 4] + (bins[:, 1] > 4) * 5)
    if n_classes == 1:
        return bins, n_bins, vals, sig * 0.37 + rng.normal(size=n), None
    y = ((sig + rng.integers(0, 2, size=n)) % n_classes).astype(np.int64)
    cnt = np.bincount(y, minlength=n_classes).astype(np.float64)
    return bins, n_bins, vals, y, (float(n) / (float(n_classes) * cnt))[y]


def forest_sha(f):
    h = hashlib.sha256()
    for k in ("baseline", "tree_seq", "tree_offset", "feature", "threshold", "missing_left", "left", "right", "value"):
        h.update(np.ascontiguousarray(f[k]).tobytes())
    return h.hexdigest()


def fit(n_classes, n, n_iter, lr=0.1, depth=5, **kw):
    bins, n_bins, vals, y, w = problem(n_classes, n)
    model = OB.train(bins, n_bins, y, n_classes, w, n_iter, lr, depth, num_leaves=15, min_data_in_leaf=10, **kw)
    return model, bins, n_bins, vals, y, w


@pytest.mark.parametrize("n_classes,n,n_iter", [(3, 1500, 12), (1, 1200, 10)])
def test_defaults_reproduce_the_plain_trainer(n_classes, n, n_iter):
    model, bins, n_bins, vals, y, w = fit(n_classes, n, n_iter)
    assert forest_sha(OG.to_flat_forest(model, vals, len(DOMS))) == PARENT_SHA[n_classes]
    explicit, *_ = fit(n_classes, n, n_iter, boosting="gbdt", reg_alpha=0.0, min_split_gain=0.0)
    assert forest_sha(OG.to_flat_forest(explicit, vals, len(DOMS))) == PARENT_SHA[n_classes]


def _leaves(model):
    return [nd for it in model["trees"] for nodes in it for nd in nodes if nd[0] < 0]


def test_huge_min_split_gain_leaves_single_leaf_trees():
    model, *_ = fit(3, 600, 5, min_split_gain=1e9)
    assert all(len(nodes) == 1 for it in model["trees"] for nodes in it)
    plain, *_ = fit(3, 600, 5)
    assert any(len(nodes) > 1 for it in plain["trees"] for nodes in it)


def test_reg_alpha_above_every_gradient_sum_zeroes_the_leaves():
    # every |G_q| <= n * max|g| * qscale, i.e. reg_alpha >= n * max weight suffices
    model, bins, n_bins, vals, y, w = fit(3, 600, 4, reg_alpha=600 * 10.0)
    assert float(w.max()) < 10.0
    assert all(nd[5] == 0.0 for nd in _leaves(model))


@pytest.mark.parametrize("reg_alpha,reg_lambda", [(0.5, 0.0), (3.0, 1.5)])
def test_reg_alpha_leaves_are_the_soft_threshold_of_their_rows(reg_alpha, reg_lambda):
    """One regression round from the initial score: every leaf is -T(G) / (H + lambda_q) * lr over the
    rows that reach it."""
    n, lr = 800, 0.3
    bins, n_bins, vals, y, _ = problem(1, n)
    model = OB.train(bins, n_bins, y, 1, None, 1, lr, 4, num_leaves=12, min_data_in_leaf=10, reg_alpha=reg_alpha,
                     reg_lambda=reg_lambda)
    init = model["init"][0]
    qscale = float(2 ** OG.quant_bits(n)) / float(np.abs(y - init).max())
    gq = np.rint((init - y) * qscale).astype(np.int64)
    hq = np.rint(np.ones(n) * qscale).astype(np.int64)
    nodes = model["trees"][0][0]
    leaf = OB.leaf_of(nodes, bins, n_bins)
    a_q, l_q = reg_alpha * qscale, reg_lambda * qscale
    assert len(nodes) > 3
    for j, nd in enumerate(nodes):
        if nd[0] >= 0:
            continue
        G, H = int(gq[leaf == j].sum()), int(hq[leaf == j].sum())
        t = np.sign(G) * max(abs(float(G)) - a_q, 0.0)
        assert nd[5] == pytest.approx(-t / (H + l_q) * lr, rel=1e-12, abs=0.0)
        assert abs(nd[5]) < abs(G / (H + l_q) * lr)         # the L1 term shrinks every leaf


def test_goss_is_gbdt_during_its_warm_up():
    lr, n_iter = 0.25, 7                     # warm-up int(1 / lr) = 4 iterations
    _, _, _, shift = OB.goss_counts(900)
    goss, *_ = fit(3, 900, n_iter, lr=lr, boosting="goss")
    gbdt, *_ = fit(3, 900, n_iter, lr=lr, quant_shift=shift)
    assert shift == 3
    assert goss["trees"][:4] == gbdt["trees"][:4]
    assert goss["trees"][4:] != gbdt["trees"][4:]


def test_goss_keeps_the_top_rows_and_their_ties():
    rng = np.random.default_rng(3)
    n = 1000
    top_k, other_k, m, _ = OB.goss_counts(n)
    thr = OB.goss_other_thr(n, top_k, other_k)
    g = rng.normal(size=(n, 2))
    h = np.ones((n, 2))
    g[:300] = 5.0                             # 300 rows tie at the largest score, top_k = 200
    kept, top = OB.goss_rows(g, h, 42, 9, top_k, thr)
    assert top_k == 200 and other_k == 100 and m == 8.0
    assert top.sum() == 300 and kept[:300].all()
    g[:300] = rng.normal(size=(300, 2))
    kept, top = OB.goss_rows(g, h, 42, 9, top_k, thr)
    assert top.sum() == top_k and kept.sum() >= top_k
    others = kept & ~top
    assert 0 < others.sum() < 3 * other_k    # about other_k / (n - top_k) of the rest


def test_dart_without_drops_is_gbdt():
    dart, *_ = fit(3, 700, 8, boosting="dart", skip_drop=1.0)
    gbdt, *_ = fit(3, 700, 8)
    assert dart["trees"] == gbdt["trees"]
    assert OB.dart_schedule(8, 0.1, 42, skip_drop=1.0) == [[]] * 8


def test_dart_drops_change_the_model():
    sched = OB.dart_schedule(10, 0.1, 42, drop_rate=0.5, skip_drop=0.0)
    assert sum(len(d) for d in sched) > 0
    dart, *_ = fit(2, 700, 10, boosting="dart", drop_rate=0.5, skip_drop=0.0)
    gbdt, *_ = fit(2, 700, 10)
    assert dart["trees"] != gbdt["trees"]


def test_rf_is_the_mean_of_trees_fitted_at_the_initial_score():
    """rf: the same trees as gbdt at learning rate 0 (gradients frozen at the initial score, same bags and
    feature subsets); each leaf is -G / (H + lambda_q) / n_iter over its in-bag rows."""
    n, n_iter, lam = 700, 6, 0.5
    bins, n_bins, vals, y, _ = problem(1, n)
    kw = dict(num_leaves=10, min_data_in_leaf=10, reg_lambda=lam, subsample=0.6, subsample_freq=1)
    rf = OB.train(bins, n_bins, y, 1, None, n_iter, 0.1, 4, boosting="rf", **kw)
    frozen = OB.train(bins, n_bins, y, 1, None, n_iter, 0.0, 4, **kw)
    strip = lambda m: [[[nd[:5] for nd in nodes] for nodes in it] for it in m["trees"]]  # noqa: E731
    assert strip(rf) == strip(frozen)
    init = rf["init"][0]
    qscale = float(2 ** OG.quant_bits(n)) / float(np.abs(y - init).max())
    gq = np.rint((init - y) * qscale).astype(np.int64)
    margin = np.full(n, init)
    for it in range(n_iter):
        nodes = rf["trees"][it][0]
        bag = OG.rows_in_bag(42, it, n, 0.6)
        leaf = OB.leaf_of(nodes, bins, n_bins)
        for j, nd in enumerate(nodes):
            if nd[0] < 0:
                rows = (leaf == j) & bag
                G, H = float(gq[rows].sum()), float(rows.sum() * int(np.rint(qscale)))
                assert nd[5] == pytest.approx(-G / (H + lam * qscale) / n_iter, rel=1e-12, abs=0.0)
        margin = margin + np.array([nd[5] for nd in nodes])[leaf]
    assert np.abs(margin - init).max() > 0.0


def test_rf_needs_sampling():
    bins, n_bins, vals, y, w = problem(3, 300)
    with pytest.raises(ValueError, match="rf needs row bagging"):
        OB.train(bins, n_bins, y, 3, w, 3, 0.1, 3, boosting="rf")
    with pytest.raises(ValueError, match="rf needs row bagging"):
        OB.train(bins, n_bins, y, 3, w, 3, 0.1, 3, boosting="rf", subsample=0.5, subsample_freq=0)
    OB.train(bins, n_bins, y, 3, w, 2, 0.1, 3, boosting="rf", colsample_bytree=0.5)


@pytest.mark.parametrize("kw", [dict(), dict(drop_rate=0.5, skip_drop=0.2), dict(drop_rate=1.0, max_drop=3, skip_drop=0.0),
                                dict(seed=7, max_drop=0)])
def test_host_dart_schedule_matches_the_oracle(kw):
    from repair import gbdt as G
    seed = kw.pop("seed", 42)
    want = OB.dart_schedule(300, 0.01, seed, **kw)
    off, flat = G.dart_schedule(300, 0.01, seed, **kw)
    got = [flat[off[i]:off[i + 1]].tolist() for i in range(300)]
    assert got == want
    assert off[-1] > 0
    if kw.get("max_drop") == 3:
        assert max(len(d) for d in want) == 3


def _binned_problem(k=600, n=5000):
    from repair.forest import first_seen
    rng = np.random.default_rng(0)
    codes = rng.integers(-1, k, size=n)
    enc = [{"attr": "a", "type": "ordinal", "categories": first_seen(codes)},
           {"attr": "b", "type": "ordinal", "categories": list(range(10))}]
    return enc, {"a": codes, "b": rng.integers(0, 10, size=n)}, {"a": k, "b": 10}


def test_max_bin_bounds_the_bins_per_feature():
    from repair import gbdt as G
    enc, codes, sizes = _binned_problem()
    default = G.bin_sample(enc, codes, sizes)
    for mb in (255, 300):                       # clamped to 255: today's binning
        got = G.bin_sample(enc, codes, sizes, max_bin=mb)
        assert np.array_equal(got[0], default[0]) and np.array_equal(got[1], default[1])
        assert all(np.array_equal(a, b) for a, b in zip(got[2], default[2]))
    assert default[1][0] == G.MAX_BINS + 1
    bins, n_bins, values = G.bin_sample(enc, codes, sizes, max_bin=16)
    assert n_bins[0] <= 16 and n_bins[1] <= 16 and n_bins[0] >= 8
    assert bins[:, 0].max() <= n_bins[0] - 1
    hi, lo = values[0]
    assert np.all(lo <= hi) and np.all(hi[:-1] < lo[1:])
    bins, n_bins, _ = G.bin_sample(enc, codes, sizes, max_bin=1)   # clamped to 2: one value bin + missing
    assert list(n_bins) == [2, 2]


def test_sklearn_models_warn_about_options_without_effect(caplog):
    from repair import train as T
    rng = np.random.default_rng(1)
    X, y = rng.normal(size=(60, 2)), rng.normal(size=60)
    opts = {"model.lgb.boosting_type": "dart", "model.lgb.min_split_gain": "0.5", "model.hp.max_evals": "1",
            "model.lgb.n_estimators": "5"}
    with caplog.at_level(logging.WARNING, logger="repair"):
        forest, _ = T.build_model(X, y, False, 0, opts)
    assert forest is not None
    msgs = [r.getMessage() for r in caplog.records if "has no effect" in r.getMessage()]
    assert len(msgs) == 1
    assert "model.lgb.boosting_type=dart" in msgs[0] and "model.lgb.min_split_gain=0.5" in msgs[0]
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger="repair"):
        T.build_model(X, y, False, 0, {"model.hp.max_evals": "1", "model.lgb.n_estimators": "5"})
    assert not [r for r in caplog.records if "has no effect" in r.getMessage()]


def test_rf_search_defaults_bag_every_tree():
    from repair import search as HS
    assert HS.search(lambda p: 0.0, 1, 5, 0, defaults=HS.RF_DEFAULTS)[0] == dict(HS.DEFAULTS, subsample=0.632,
                                                                               subsample_freq=1)
    assert HS.search(lambda p: 0.0, 1, 5, 0)[0] == HS.DEFAULTS
    seen = []
    HS.search(lambda p: seen.append(dict(p)) or 1.0, 3, 5, 0, defaults=HS.RF_DEFAULTS)
    assert seen[0] == HS.RF_DEFAULTS
