"""dr_gbdt_train_ex (model.lgb.boosting_type dart / goss / rf, reg_alpha, min_split_gain, max_bin) against its
specification oracle/gbdt_boost.py, bit for bit, and through the public API."""
import os

import numpy as np
import pandas as pd
import pytest

import parity_utils as PU
from conftest import GOLDEN
from test_gbdt_options_cpu import _binned_problem, problem

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    from repair._native import Context
    c = Context(0)
    yield c
    c.close()


def _assert_same(got, want):
    for k in ("tree_seq", "tree_offset", "feature", "missing_left", "left", "right"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
    assert np.array_equal(got["threshold"], want["threshold"])
    assert np.array_equal(got["value"], want["value"])          # bit-exact float64 leaves
    assert np.array_equal(got["baseline"], want["baseline"])


def _both(ctx, bins, n_bins, vals, y, n_classes, w, n_iter, lr, depth, **kw):
    from oracle import gbdt_boost as OB
    from repair import gbdt as PG
    wt = w if w is not None else np.ones(len(y))
    want = OB.to_flat_forest(OB.train(bins, n_bins, y, n_classes, w, n_iter, lr, depth, **kw), vals, len(n_bins))
    got = PG.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, vals, y, n_classes, wt, n_iter, lr, depth, **kw)
    return got, want


MODES = {
    "gbdt": dict(reg_alpha=0.7, min_split_gain=0.02),
    "dart": dict(boosting="dart", drop_rate=0.5, skip_drop=0.1),
    "goss": dict(boosting="goss"),                  # lr 0.25: sampling from iteration 4 on
    "rf": dict(boosting="rf", subsample=0.7, subsample_freq=1),
}


@pytest.mark.parametrize("n_classes", [1, 2, 4])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_boosting_types_match_oracle_bit_for_bit(ctx, mode, n_classes):
    bins, n_bins, vals, y, w = problem(n_classes, 700)
    got, want = _both(ctx, bins, n_bins, vals, y, n_classes, w, 9, 0.25, 5, num_leaves=15, min_data_in_leaf=10,
                      **MODES[mode])
    _assert_same(got, want)
    assert (np.asarray(want["feature"]) >= 0).sum() > 9


@pytest.mark.parametrize("n_classes,kw", [
    (3, dict(reg_alpha=2.0)), (2, dict(min_split_gain=0.5)), (1, dict(reg_alpha=0.3, min_split_gain=0.05)),
    (3, dict(reg_alpha=1.0, reg_lambda=1.5, colsample_bytree=0.5, subsample=0.7, subsample_freq=2)),
    (5, dict(min_split_gain=0.2, reg_lambda=4.0, colsample_bytree=0.3, subsample=0.6, subsample_freq=1,
             num_leaves=32)),
    (2, dict(reg_alpha=0.5, min_split_gain=0.1, reg_lambda=0.3, subsample=0.8, subsample_freq=1))])
def test_l1_and_gain_floor_match_oracle_bit_for_bit(ctx, n_classes, kw):
    bins, n_bins, vals, y, w = problem(n_classes, 900)
    args = dict(num_leaves=15, min_data_in_leaf=10)
    args.update(kw)
    got, want = _both(ctx, bins, n_bins, vals, y, n_classes, w, 7, 0.1, 5, **args)
    _assert_same(got, want)


def test_goss_with_ties_at_the_threshold_matches_oracle(ctx):
    """Learning rate 1: sampling from iteration 1 on, when every row of a leaf and class has the same score,
    so hundreds of rows tie at the top_k-th largest."""
    from oracle import gbdt_boost as OB
    bins, n_bins, vals, y, w = problem(2, 800)
    kw = dict(num_leaves=6, min_data_in_leaf=10, boosting="goss")
    got, want = _both(ctx, bins, n_bins, vals, y, 2, w, 6, 1.0, 3, **kw)
    _assert_same(got, want)
    # the tie is real: at iteration 1 the row scores take few distinct values
    first = OB.train(bins, n_bins, y, 2, w, 1, 1.0, 3, num_leaves=6, min_data_in_leaf=10)
    nodes = first["trees"][0][0]
    assert len(set(OB.leaf_of(nodes, bins, n_bins).tolist())) <= 6


@pytest.mark.parametrize("kw", [dict(drop_rate=1.0, max_drop=2, skip_drop=0.0), dict(drop_rate=0.3, skip_drop=0.3)])
def test_dart_drops_match_oracle_bit_for_bit(ctx, kw):
    from oracle import gbdt_boost as OB
    bins, n_bins, vals, y, w = problem(3, 800)
    sched = OB.dart_schedule(10, 0.2, 42, **kw)
    assert sum(map(len, sched)) > 3
    if kw.get("max_drop") == 2:
        assert max(map(len, sched)) == 2
    got, want = _both(ctx, bins, n_bins, vals, y, 3, w, 10, 0.2, 4, num_leaves=12, min_data_in_leaf=10,
                      boosting="dart", **kw)
    _assert_same(got, want)


@pytest.mark.parametrize("kw", [dict(subsample=0.6, subsample_freq=2), dict(colsample_bytree=0.5)])
def test_rf_matches_oracle_bit_for_bit(ctx, kw):
    bins, n_bins, vals, y, w = problem(3, 800)
    got, want = _both(ctx, bins, n_bins, vals, y, 3, w, 8, 0.1, 5, num_leaves=15, min_data_in_leaf=10,
                      boosting="rf", **kw)
    _assert_same(got, want)


def test_rf_without_sampling_is_refused(ctx):
    from repair._native import NativeError
    from repair import gbdt as PG
    bins, n_bins, vals, y, w = problem(2, 300)
    with pytest.raises(NativeError, match="invalid argument: boosting rf needs row bagging"):
        PG.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, vals, y, 2, w, 3, 0.1, 3, boosting="rf")


@pytest.mark.parametrize("max_bin", [2, 16, 255])
def test_max_bin_on_a_600_value_feature_matches_oracle(ctx, max_bin):
    from repair import gbdt as PG
    enc, codes, sizes = _binned_problem()
    bins, n_bins, values = PG.bin_sample(enc, codes, sizes, max_bin=max_bin)
    assert 2 <= n_bins[0] <= max_bin and (max_bin != 255 or n_bins[0] == 255)
    rng = np.random.default_rng(max_bin)
    y = ((bins[:, 0].astype(np.int64) * 7 // max(int(n_bins[0]), 1) + bins[:, 1] + rng.integers(0, 2, len(bins))) % 3)
    y[:3] = [0, 1, 2]                            # every class present
    w = PG.class_weights(y, 3, True)
    # a grouped feature's bin values are (largest, smallest) per bin, which oracle/gbdt.py's flattening does not
    # take: it flattens with bin value = bin index, and the split bins it records give the expected thresholds
    index = [np.arange(256, dtype=np.float64)] * bins.shape[1]
    _, want = _both(ctx, bins, n_bins, index, y, 3, w, 5, 0.1, 5, num_leaves=15, min_data_in_leaf=10, reg_alpha=0.1)
    inner = np.asarray(want["feature"]) >= 0
    t = np.floor(want["threshold"][inner]).astype(np.int64)
    hi_lo = [(v, v) if np.ndim(v) == 1 else (v[0], v[1]) for v in values]
    want["threshold"][inner] = [(hi_lo[f][0][b] + hi_lo[f][1][b + 1]) / 2.0
                                for f, b in zip(np.asarray(want["feature"])[inner], t)]
    got = PG.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, values, y, 3, w, 5, 0.1, 5, num_leaves=15,
                       min_data_in_leaf=10, reg_alpha=0.1)
    _assert_same(got, want)
    if max_bin > 2:
        assert inner.sum() > 5 and (np.asarray(want["feature"])[inner] == 0).any()


def _raw(ctx, bins, n_bins, y, w, n_classes, n_iter, boost, ex):
    from repair import gbdt as PG
    from repair._native import dr_gbdt_params
    n, F = bins.shape
    S = 1 if n_classes <= 2 else n_classes
    init = PG.initial_scores(y, n_classes, w)
    prm = dr_gbdt_params(n, F, n_classes, n_iter, 5, 15, 10, 0.1, 1e-3, float(2 ** PG.quant_bits(n)) / float(w.max()),
                         0.5, 0.8, 0.7, 2, 42)
    dev = torch.device("cuda", 0)
    d_bins = torch.from_numpy(bins).to(dev)
    d_y = torch.from_numpy(np.ascontiguousarray(y, dtype=np.int32)).to(dev)
    d_w = torch.from_numpy(np.ascontiguousarray(w, dtype=np.float64)).to(dev)
    ws = torch.full((ctx.gbdt_workspace_bytes(n, S),), 7, dtype=torch.uint8, device=dev)
    nodes = torch.zeros(n_iter * S * PG.MAX_NODES * PG.NODE_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    counts = torch.zeros(n_iter * S, dtype=torch.int32, device=dev)
    before = ctx.launch_count
    if ex:
        ctx.gbdt_train_ex(prm, boost, d_bins, n_bins, d_y, None, d_w, init, ws, nodes, counts)
    else:
        ctx.gbdt_train(prm, d_bins, n_bins, d_y, None, d_w, init, ws, nodes, counts)
    return nodes.cpu().numpy().tobytes(), counts.cpu().numpy().tobytes(), ctx.launch_count - before


def test_train_ex_at_defaults_is_dr_gbdt_train_byte_for_byte(ctx):
    from repair._native import dr_gbdt_boost
    bins, n_bins, vals, y, w = problem(3, 1000)
    want = _raw(ctx, bins, n_bins, y, w, 3, 6, None, False)
    assert _raw(ctx, bins, n_bins, y, w, 3, 6, None, True) == want
    explicit = dr_gbdt_boost(0, 0, 0, 0, 0.0, 0.0, None, None)       # gbdt, no L1, no gain floor
    assert _raw(ctx, bins, n_bins, y, w, 3, 6, explicit, True) == want


# ---- through the public API ----------------------------------------------------------------------------
ADULT_OPTS = {"model.hp.max_evals": 1, "model.lgb.n_estimators": 300}


def _adult(**opts):
    adult = pd.read_csv(os.path.join(GOLDEN, "adult.csv"))
    return PU.run_product(adult, "tid", [{"type": "null"}], opts=dict(ADULT_OPTS, **opts))


def _gpu_forests(rm):
    out = []
    for _, m in rm.last_run["models"]:
        if m[0] != "forest":
            continue
        c = m[2]["ctx"]
        if c["is_discrete"] and all(e["type"] != "cont" for e in c["encoders"]):
            out.append((m[2]["spec"]["forest"], c))
    assert out
    return out


@pytest.mark.parametrize("boosting", ["dart", "goss", "rf"])
def test_every_boosting_type_repairs_adult(boosting):
    rm, out = _adult(**{"model.lgb.boosting_type": boosting})
    base_rm, base = _adult()
    assert list(out.columns) == list(base.columns)
    assert sorted((g[0], g[1]) for g in PU.frame_tuples(out, "tid")) == \
        sorted((g[0], g[1]) for g in PU.frame_tuples(base, "tid"))
    assert len(_gpu_forests(rm)) == len(_gpu_forests(base_rm))


def test_huge_min_split_gain_leaves_no_split():
    rm, _ = _adult(**{"model.lgb.min_split_gain": 1e9, "model.lgb.reg_alpha": 0.5})
    for forest, _ in _gpu_forests(rm):
        assert (np.asarray(forest["feature"]) < 0).all()


def test_rf_leaves_are_a_300th_of_the_unscaled_fits():
    """Every tree of an rf model is its unscaled fit -G / H at the initial score over its bag (trial 0:
    subsample 0.632 every iteration), divided by n_estimators."""
    from oracle import gbdt as OG
    from repair import gbdt as PG
    rm, _ = _adult(**{"model.lgb.boosting_type": "rf"})
    for forest, c in _gpu_forests(rm):
        yv = np.asarray(c["y_values"])
        classes = sorted(set(yv.tolist()))
        yi = np.searchsorted(np.asarray(classes), yv)
        n, C = len(yi), len(classes)
        w = PG.class_weights(yi, C, True)
        init = PG.initial_scores(yi, C, w)
        qscale = float(2 ** PG.quant_bits(n)) / float(w.max())
        S = 1 if C <= 2 else C
        if C == 2:
            p = OG.sigmoid_det(np.full(n, init[0]))[:, None]
            g, h = (p[:, 0] - yi) * w, p[:, 0] * (1.0 - p[:, 0]) * w
            g, h = g[:, None], h[:, None]
        else:
            p = OG.softmax_det(np.tile(init, (n, 1)))
            onehot = np.eye(C)[yi]
            g, h = (p - onehot) * w[:, None], float(S) / float(S - 1) * p * (1.0 - p) * w[:, None]
        gq, hq = np.rint(g * qscale).astype(np.int64), np.rint(h * qscale).astype(np.int64)
        off = np.asarray(forest["tree_offset"])
        assert (np.asarray(forest["feature"]) < 0).all()            # 20 rows: no leaf may split
        for t in range(len(off) - 1):
            it, s = t // S, t % S
            bag = OG.rows_in_bag(42, it, n, 0.632)
            G, H = float(gq[bag, s].sum()), float(hq[bag, s].sum())
            want = -(G / H) / 300.0 if H > 0 else 0.0
            assert forest["value"][off[t]] == want


def test_explicit_default_options_leave_the_forests_unchanged():
    base, _ = _adult()
    explicit, _ = _adult(**{"model.lgb.boosting_type": "gbdt", "model.lgb.reg_alpha": 0.0,
                            "model.lgb.min_split_gain": 0.0, "model.lgb.max_bin": 255})
    a, b = _gpu_forests(base), _gpu_forests(explicit)
    assert len(a) == len(b)
    for (fa, _), (fb, _) in zip(a, b):
        for k in fa:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), k
