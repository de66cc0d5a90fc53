"""Continuous targets and features in the GPU trainer: dr_gbdt_train(_ex) on quantile-binned columns against
oracle/gbdt_boost.py bit for bit, and models with a continuous target or feature under
model.lgb.boosting_type / reg_alpha / min_split_gain through the public API on boston and iris."""
import logging
import math
import os

import numpy as np
import pandas as pd
import pytest

import parity_utils as PU
from conftest import GOLDEN

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


def _oracle(bins, n_bins, values, y, n_classes, w, n_iter, lr, depth, **kw):
    """oracle/gbdt_boost.py's forest with thresholds in value space: midway between the split bin's largest
    and the next bin's smallest value.  These plain midpoints skip gbdt.flatten's fallback for infinite or
    adjacent values, which is sound only because the problems here are finite and rounded (the fallback has
    its own CPU tests).  A regression runs on its target scaled by 2^-k (gbdt.regression_scale), with
    reg_alpha * 2^-k and min_split_gain * 2^-2k, and its leaves and baseline are scaled back by 2^k."""
    from oracle import gbdt_boost as OB
    from repair import gbdt as G
    k = 0
    if n_classes == 1:
        goss_shift = OB.goss_counts(len(y))[3] if kw.get("boosting") == "goss" else 0
        k = G.regression_scale(y, G.initial_scores(y, 1, None)[0], len(y), goss_shift)
        y = np.ldexp(np.asarray(y, dtype=np.float64), -k)
        kw = dict(kw, reg_alpha=float(np.ldexp(kw.get("reg_alpha", 0.0), -k)),
                  min_split_gain=float(np.ldexp(kw.get("min_split_gain", 0.0), -2 * k)))
    model = OB.train(bins, n_bins, y, n_classes, w, n_iter, lr, depth, **kw)
    want = OB.to_flat_forest(model, [np.arange(256, dtype=np.float64)] * len(n_bins), len(n_bins))
    want["baseline"], want["value"] = np.ldexp(want["baseline"], k), np.ldexp(want["value"], k)
    inner = np.asarray(want["feature"]) >= 0
    hi_lo = [(v, v) if np.ndim(v) == 1 else (v[0], v[1]) for v in values]
    want["threshold"][inner] = [(hi_lo[f][0][b] + hi_lo[f][1][b + 1]) / 2.0 for f, b in
                                zip(np.asarray(want["feature"])[inner], np.floor(want["threshold"][inner]).astype(int))]
    return want


def cont_problem(n_classes, n, seed=3):
    """Quantile-binned continuous columns: a > 254-value column, NULLs, a duplicate-heavy column, and one
    discrete (ordinal) column beside them."""
    from repair import gbdt as G
    rng = np.random.default_rng(seed)
    x = {"wide": np.round(rng.normal(size=n) * 50.0, 3),
         "nulls": np.where(rng.random(n) < 0.25, np.nan, np.round(rng.uniform(0, 10, size=n), 1)),
         "dup": rng.choice([-1.5, 0.25, 3.0, 8.0], size=n),
         "small": np.round(rng.normal(size=n), 2)}
    x["wide"][rng.random(n) < 0.05] = np.nan
    codes = rng.integers(0, 6, size=n)
    enc = [{"attr": a, "type": "cont"} for a in x] + [{"attr": "d", "type": "ordinal", "categories": list(range(6))}]
    bins, n_bins, values = G.bin_sample(enc, {"d": codes}, {"d": 6}, sample_values=x)
    sig = np.nan_to_num(x["wide"]) / 40.0 + np.nan_to_num(x["nulls"], nan=12.0) / 3.0 + (x["dup"] > 1) * 2 + codes * 0.5
    if n_classes == 1:
        return bins, n_bins, values, sig + rng.normal(size=n) * 0.3, None
    if n_classes == 0:                            # regression with a spread below 1: scaled up
        return bins, n_bins, values, (sig + rng.normal(size=n) * 0.3) * 0.01, None
    if n_classes == -1:                           # price-sized regression: scaled down
        return bins, n_bins, values, (sig + rng.normal(size=n) * 0.3) * 4.0e4 + 2.0e5, None
    y = (np.floor(sig + rng.normal(size=n) * 0.5).astype(np.int64) % n_classes)
    return bins, n_bins, values, y, G.class_weights(y, n_classes, True)


MODES = {
    "gbdt_l1_gain": dict(reg_alpha=0.7, min_split_gain=0.02),
    "dart": dict(boosting="dart", drop_rate=0.5, skip_drop=0.1),
    "goss": dict(boosting="goss"),
    "rf": dict(boosting="rf", subsample=0.7, subsample_freq=1),
}


@pytest.mark.parametrize("n_classes", [0, 1, 2, 4])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_continuous_bins_match_oracle_bit_for_bit(ctx, mode, n_classes):
    from repair import gbdt as G
    bins, n_bins, values, y, w = cont_problem(n_classes, 900)
    assert n_bins[0] == 255 and np.ndim(values[0]) == 2                    # the > 254-value column is grouped
    C = max(n_classes, 1)
    kw = dict(num_leaves=15, min_data_in_leaf=10, **MODES[mode])
    want = _oracle(bins, n_bins, values, y, C, w, 9, 0.25, 5, **kw)
    got = G.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, values, y, C,
                      w if w is not None else np.ones(len(y)), 9, 0.25, 5, **kw)
    _assert_same(got, want)
    assert (np.asarray(want["feature"]) >= 0).sum() > 9
    assert {0, 1} <= set(np.asarray(want["feature"]).tolist())              # splits on the continuous columns


@pytest.mark.parametrize("mode", ["goss", "gbdt_l1_gain"])
def test_price_sized_regression_keeps_its_hessian_precision(ctx, mode):
    """A target of price magnitude on 8 193+ rows (quantisation width 16 bits): unscaled, its spread of a
    few 1e5 would quantise every row's hessian to 0 and no tree would split.  Scaled, it matches the oracle
    bit for bit, splits, and beats filling with the mean on held-out rows."""
    from oracle import gbdt_boost as OB
    from oracle.forest import forest_predict
    from repair import gbdt as G
    n = 11000
    bins, n_bins, values, y, _ = cont_problem(-1, n)
    tr, te = np.arange(n) < 9000, np.arange(n) >= 9000
    init = G.initial_scores(y[tr], 1, None)[0]
    goss_shift = OB.goss_counts(int(tr.sum()))[3] if mode == "goss" else 0
    assert G.quant_bits(int(tr.sum())) == 16
    assert np.rint(2.0 ** 16 / np.abs(y[tr] - init).max()) == 0.0       # unscaled: every hessian would be 0
    k = G.regression_scale(y[tr], init, int(tr.sum()), goss_shift)
    assert k > 0 and 1.0 <= np.ldexp(np.abs(y[tr] - init).max(), -k) < 2.0
    kw = dict(num_leaves=15, min_data_in_leaf=10, **MODES[mode])
    b = np.ascontiguousarray(bins[tr])
    want = _oracle(b, n_bins, values, y[tr], 1, None, 9, 0.25, 5, **kw)
    got = G.train_gpu(ctx, torch.device("cuda", 0), b, n_bins, values, y[tr], 1, np.ones(int(tr.sum())), 9, 0.25,
                      5, **kw)
    _assert_same(got, want)
    assert (np.asarray(got["feature"]) >= 0).sum() > 50
    # held-out rows: predict from the binned values (the bin's smallest value lies on its side of every split)
    lo = [v if np.ndim(v) == 1 else v[1] for v in values]
    X = np.stack([np.where(bins[te, f] == n_bins[f] - 1, np.nan, np.asarray(lo[f])[np.minimum(bins[te, f],
                  len(lo[f]) - 1)]) for f in range(len(n_bins))], axis=1)
    mse = float(np.mean((forest_predict(got, X) - y[te]) ** 2))
    mse_mean = float(np.mean((init - y[te]) ** 2))
    assert mse < 0.8 * mse_mean, (mse, mse_mean)


# ---- through the public API ----------------------------------------------------------------------------
def boston_bin():
    df = pd.read_csv(os.path.join(GOLDEN, "bin_boston.csv"))
    df["CHAS"] = df["CHAS"].map(lambda v: None if v != v else str(v))
    df["RAD"] = df["RAD"].map(lambda v: None if v != v else str(int(v)) if float(v).is_integer() else str(v))
    for c in ("ZN", "TAX"):
        df[c] = df[c].astype("Int64")
    return df


def _boston(caplog, mode="repair", given=None, **opts):
    with caplog.at_level(logging.WARNING, logger="repair"):
        rm, out = PU.run_product(boston_bin(), "tid", [{"type": "null"}], opts=opts, mode=mode, given=given)
    assert not [r for r in caplog.records if "has no effect" in r.getMessage()]
    caplog.clear()
    return rm, out


def _cont_models(rm):
    out = []
    for y, m in rm.last_run["models"]:
        if m[0] != "forest":
            continue
        c = m[2]["ctx"]
        if not c["is_discrete"] or any(e["type"] == "cont" for e in c["encoders"]):
            out.append((y, m[2]["spec"]["forest"], c))
    assert out
    return out


def _rebin(c, dict_sizes, max_bin):
    """The model's training context binned again from its encoded matrix X.  This goes through gbdt.bin_column,
    the code that binned the model, so the end-to-end comparison below checks the trainer, the routing and the
    regression conventions, not the binning: tests/test_gbdt_cont_cpu.py checks the bins on their own."""
    from repair import gbdt as G
    from repair.forest import encoder_lut
    X, j, parts = np.asarray(c["X"], dtype=np.float64), 0, []
    for e in c["encoders"]:
        if e["type"] == "cont":
            doms = [np.unique(X[~np.isnan(X[:, j]), j])]
        else:
            lut = encoder_lut(e, dict_sizes[e["attr"]])
            doms = [np.unique(lut[~np.isnan(lut[:, k]), k]) for k in range(lut.shape[1])]
        for d in doms:
            parts.append(G.bin_column(X[:, j], d, min(255, max_bin) - 1))
            j += 1
    return (np.stack([p[0] for p in parts], axis=1), np.array([p[1] for p in parts], dtype=np.int32),
            [p[2] for p in parts])


def _dict_sizes():
    from repair.table import EncodedTable
    return {c.name: c.dict_size for c in EncodedTable.from_pandas(boston_bin(), "tid").columns}


N_EST, LR = 40, 0.1
API_MODES = {"dart": {"model.lgb.boosting_type": "dart"}, "goss": {"model.lgb.boosting_type": "goss"},
             "rf": {"model.lgb.boosting_type": "rf"},
             "l1_gain": {"model.lgb.reg_alpha": 0.5, "model.lgb.min_split_gain": 0.01}}


@pytest.mark.parametrize("mode", sorted(API_MODES))
def test_boston_continuous_models_equal_the_oracle(caplog, mode):
    from repair import gbdt as G
    from repair import search as HS
    opts = dict(API_MODES[mode], **{"model.lgb.n_estimators": N_EST, "model.lgb.learning_rate": LR})
    rm, _ = _boston(caplog, **opts)
    sizes = _dict_sizes()
    models = _cont_models(rm)
    assert {y for y, _, _ in models} == {"CRIM", "RAD", "TAX", "LSTAT"}
    params = HS.RF_DEFAULTS if mode == "rf" else HS.DEFAULTS
    for y, forest, c in models:
        bins, n_bins, values = _rebin(c, sizes, 255)
        yv = np.asarray(c["y_values"])
        if c["is_discrete"]:
            classes = sorted(set(int(v) for v in yv.tolist()))
            yf = np.searchsorted(np.asarray(classes), yv)
            C, w = len(classes), G.class_weights(yf, len(classes), True)
        else:
            yf, C, w = yv.astype(np.float64), 1, None
        want = _oracle(bins, n_bins, values, yf, C, w, N_EST, LR, 7, num_leaves=31, min_data_in_leaf=20,
                       min_sum_hessian=1e-3, reg_lambda=0.0, colsample_bytree=1.0, subsample=params["subsample"],
                       subsample_freq=params["subsample_freq"],
                       boosting=API_MODES[mode].get("model.lgb.boosting_type", "gbdt"),
                       reg_alpha=API_MODES[mode].get("model.lgb.reg_alpha", 0.0),
                       min_split_gain=API_MODES[mode].get("model.lgb.min_split_gain", 0.0))
        _assert_same(forest, want)


@pytest.fixture(scope="module")
def boston_default():
    return PU.run_product(boston_bin(), "tid", [{"type": "null"}])


def _cells(out):
    return sorted((int(t), a) for t, a in zip(out["tid"], out["attribute"]))


@pytest.mark.parametrize("mode", ["dart", "goss", "rf", "l1_gain"])
def test_boston_repairs_the_same_cells_and_beats_the_mean(caplog, boston_default, mode):
    rm, out = _boston(caplog, **API_MODES[mode])
    base_rm, base = boston_default
    assert _cells(out) == _cells(base)
    if mode == "l1_gain":
        return
    clean = pd.read_csv(os.path.join(GOLDEN, "boston_clean.csv"), dtype=str)
    clean["tid"] = clean["tid"].astype(int)
    rep = out[["tid", "attribute", "repaired"]].copy()
    rep["tid"] = rep["tid"].astype(int)
    cmp = rep.merge(clean, on=["tid", "attribute"], how="inner")
    mean = {y: float(np.mean(c["y_values"])) for y, _, c in _cont_models(rm)}
    for a in ("CRIM", "LSTAT", "TAX"):
        sel = cmp[cmp.attribute == a]
        truth = pd.to_numeric(sel["correct_val"]).to_numpy(dtype=np.float64)
        got = pd.to_numeric(sel["repaired"]).to_numpy(dtype=np.float64)
        assert len(sel) > 20
        rmse = math.sqrt(float(np.mean((truth - got) ** 2)))
        base_rmse = math.sqrt(float(np.mean((truth - mean[a]) ** 2)))
        assert rmse < base_rmse, (a, rmse, base_rmse)


def test_default_options_keep_scikit_learn_for_continuous_models(boston_default):
    from repair.train import build_model
    rm, _ = boston_default
    for y, forest, c in _cont_models(rm):
        want, classes = build_model(c["X"], c["y_values"], c["is_discrete"], c["num_class"], c["opts"])
        for k in want:
            assert np.array_equal(np.asarray(forest[k]), np.asarray(want[k])), (y, k)


def test_goss_search_runs_cross_validation_on_the_device(caplog):
    with caplog.at_level(logging.WARNING, logger="repair"):
        rm, out = PU.run_product(pd.read_csv(os.path.join(GOLDEN, "iris.csv")), "tid", [{"type": "null"}],
                                 opts={"model.lgb.boosting_type": "goss", "model.hp.max_evals": 3,
                                       "model.lgb.n_estimators": 60})
    assert not [r for r in caplog.records if "has no effect" in r.getMessage() or "class 'ValueError'"
                in r.getMessage()]
    assert len(out) > 0
    targets = [y for y, m in rm.last_run["models"] if m[0] == "forest"]
    assert sorted(targets) == ["petal_length", "petal_width", "sepal_length", "sepal_width"]
    for y in targets:
        assert rm.last_run["search"][y]["evals"] == 3


def test_huge_min_split_gain_leaves_continuous_models_without_splits(caplog):
    rm, _ = _boston(caplog, **{"model.lgb.min_split_gain": 1e9, "model.lgb.n_estimators": 20})
    for _, forest, _ in _cont_models(rm):
        assert (np.asarray(forest["feature"]) < 0).all()


def test_candidate_probabilities_under_goss(caplog):
    df = boston_bin()
    given = pd.DataFrame({"tid": list(range(20)) + df.tid[df.RAD.isna()].tolist(),
                          "attribute": ["CHAS"] * 20 + ["RAD"] * int(df.RAD.isna().sum())})
    rm, out = _boston(caplog, mode="pmf", given=given,
                      **{"model.lgb.boosting_type": "goss", "model.lgb.n_estimators": 60})
    for a in ("CHAS", "RAD"):
        sel = out[out.attribute == a]
        assert len(sel) > 0
        for pmf in sel["pmf"]:
            assert pmf and all(0.0 < p["prob"] <= 1.0 for p in pmf)
    forests = {y for y, _, _ in _cont_models(rm)}
    assert {"CHAS", "RAD"} <= forests
