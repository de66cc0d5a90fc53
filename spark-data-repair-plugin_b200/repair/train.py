"""Repair-model producer.

The reference trains LightGBM 3.3.1 under a hyperopt TPE search (``train.py:89-229``); neither
package is available offline, and SURVEY.md section 8 keeps training out of the first bar (the model
is *consumed* by the hot path).  This module produces the same kind of object -- a gradient-boosted
forest with the reference's fixed parameters -- with scikit-learn's histogram GBDT and flattens
it into the exchange format of ``forest.py``.  Training parity with LightGBM is therefore
UNPINNED (DESIGN.md); inference parity is exact for whatever forest is handed over.
"""
import logging

import numpy as np

from .utils import get_option_value

_logger = logging.getLogger("repair")

# option keys accepted for API compatibility with train.py:36-86 (key, default, type, validator, message)
_OPTS = [
    ("model.lgb.boosting_type", "gbdt", str, lambda v: v in ["gbdt", "dart", "goss", "rf"],
     "`{}` should be in ['gbdt', 'dart', 'goss', 'rf']"),
    ("model.lgb.class_weight", "balanced", str, None, None),
    ("model.lgb.learning_rate", 0.01, float, lambda v: v > 0.0, "`{}` should be positive"),
    ("model.lgb.max_depth", 7, int, None, None),
    ("model.lgb.max_bin", 255, int, None, None),
    ("model.lgb.reg_alpha", 0.0, float, lambda v: v >= 0.0, "`{}` should be greater than or equal to 0.0"),
    ("model.lgb.min_split_gain", 0.0, float, lambda v: v >= 0.0, "`{}` should be greater than or equal to 0.0"),
    ("model.lgb.n_estimators", 300, int, lambda v: v > 0, "`{}` should be positive"),
    ("model.lgb.importance_type", "gain", str, lambda v: v in ["split", "gain"], "`{}` should be in ['split', 'gain']"),
    ("model.cv.n_splits", 3, int, lambda v: v >= 3, "`{}` should be greater than 2"),
    ("model.hp.timeout", 0, int, None, None),
    ("model.hp.max_evals", 100000000, int, lambda v: v > 0, "`{}` should be positive"),
    ("model.hp.no_progress_loss", 50, int, lambda v: v > 0, "`{}` should be positive"),
]
train_option_keys = [o[0] for o in _OPTS]
_OPT = {o[0]: o for o in _OPTS}


def _get(opts, key):
    return get_option_value(opts, *_OPT[key])


def validate_options(opts):
    for key in train_option_keys:
        _get(opts, key)


def flatten_sklearn(est, n_features, n_classes):
    """HistGradientBoosting{Classifier,Regressor} -> flat forest (numerical splits only)."""
    feature, threshold, missing_left, left, right, value = [], [], [], [], [], []
    tree_seq, tree_offset = [], [0]
    for per_iter in est._predictors:
        for s, pred in enumerate(per_iter):
            nd = pred.nodes
            if nd["is_categorical"].any():
                raise ValueError("categorical splits are not part of the exchange format")
            leaf = nd["is_leaf"].astype(bool)
            feature.append(np.where(leaf, -1, nd["feature_idx"]).astype(np.int32))
            threshold.append(np.where(leaf, 0.0, nd["num_threshold"]).astype(np.float64))
            missing_left.append(nd["missing_go_to_left"].astype(np.uint8))
            left.append(np.where(leaf, 0, nd["left"]).astype(np.int32))
            right.append(np.where(leaf, 0, nd["right"]).astype(np.int32))
            value.append(np.where(leaf, nd["value"], 0.0).astype(np.float64))
            tree_seq.append(s)
            tree_offset.append(tree_offset[-1] + len(nd))
    cat = (lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dtype=dt))
    return {
        "n_features": int(n_features), "n_classes": int(n_classes),
        "baseline": np.asarray(est._baseline_prediction, dtype=np.float64).reshape(-1).copy(),
        "tree_seq": np.asarray(tree_seq, dtype=np.int32), "tree_offset": np.asarray(tree_offset, dtype=np.int64),
        "feature": cat(feature, np.int32), "threshold": cat(threshold, np.float64),
        "missing_left": cat(missing_left, np.uint8), "left": cat(left, np.int32), "right": cat(right, np.int32),
        "value": cat(value, np.float64),
    }


def search_options(opts):
    """(max_evals, no_progress_loss, timeout, n_splits) of train.py:72-86."""
    return (_get(opts, "model.hp.max_evals"), _get(opts, "model.hp.no_progress_loss"), _get(opts, "model.hp.timeout"),
            _get(opts, "model.cv.n_splits"))


def sklearn_estimator(is_discrete, opts, params):
    """scikit-learn histogram GBDT with the reference's fixed parameters (train.py:102-115) and the tuned
    ones it has a counterpart for: num_leaves -> max_leaf_nodes, min_child_samples -> min_samples_leaf,
    reg_lambda -> l2_regularization, colsample_bytree -> max_features (per split instead of per tree);
    min_child_weight and row sub-sampling have no counterpart and are ignored."""
    from sklearn.ensemble import HistGradientBoostingClassifier, HistGradientBoostingRegressor
    common = dict(
        learning_rate=_get(opts, "model.lgb.learning_rate"),
        max_iter=_get(opts, "model.lgb.n_estimators"),
        max_depth=_get(opts, "model.lgb.max_depth") if _get(opts, "model.lgb.max_depth") > 0 else None,
        max_leaf_nodes=max(2, int(params["num_leaves"])), min_samples_leaf=max(1, int(params["min_child_samples"])),
        max_bins=min(255, max(2, _get(opts, "model.lgb.max_bin"))),
        l2_regularization=float(params["reg_lambda"]), early_stopping=False, random_state=42)
    try:
        import inspect
        if "max_features" in inspect.signature(HistGradientBoostingRegressor.__init__).parameters:
            common["max_features"] = float(min(1.0, max(params["colsample_bytree"], 1e-3)))
    except (TypeError, ValueError):
        pass
    if is_discrete:
        cw = _get(opts, "model.lgb.class_weight")
        return HistGradientBoostingClassifier(class_weight="balanced" if cw == "balanced" else None, **common)
    return HistGradientBoostingRegressor(**common)


# model.lgb.* options scikit-learn's histogram GBDT has no counterpart for, with their defaults
_GPU_ONLY_OPTS = (("model.lgb.boosting_type", "gbdt"), ("model.lgb.reg_alpha", 0.0), ("model.lgb.min_split_gain", 0.0))


def build_model(X, y, is_discrete, num_class, opts):
    """-> (flat forest, class labels ascending or None) or (None, None) when training fails
    (the reference swallows failures into PoorModel(None), train.py:227-229).

    Fixed parameters follow train.py:102-115; the seven tuned parameters come from the search of
    search.py (train.py:133-229) -- LightGBM's defaults when ``model.hp.max_evals`` is 1."""
    from . import search as HS
    ignored = ["{}={}".format(k, _get(opts, k)) for k, d in _GPU_ONLY_OPTS if _get(opts, k) != d]
    if ignored:
        _logger.warning("{} has no effect on this model: it is trained by scikit-learn's histogram GBDT "
                        "(continuous target or features), which has no dart, goss, rf, L1 or gain floor"
                        .format(", ".join(ignored)))
    try:
        X = np.asarray(X, dtype=np.float64)
        if X.shape[1] == 0:
            X = np.zeros((X.shape[0], 1))
        yv = np.asarray(y) if is_discrete else np.asarray(y, dtype=np.float64)
        max_evals, no_progress, timeout, n_splits = search_options(opts)
        folds = HS.cv_folds(yv, is_discrete, n_splits) if max_evals > 1 else None

        def evaluate(params):
            scores = []
            for tr, va in folds:
                est = sklearn_estimator(is_discrete, opts, params)
                est.fit(X[tr], yv[tr])
                scores.append(HS.score(yv[va], est.predict(X[va]), is_discrete))
            return -float(np.mean(scores)), [-float(v) for v in scores]

        params, _, _ = HS.search(evaluate, max_evals, no_progress, timeout)
        est = sklearn_estimator(is_discrete, opts, params)
        est.fit(X, yv)
        if is_discrete:
            classes = [c.item() if hasattr(c, "item") else c for c in est.classes_]
            return flatten_sklearn(est, X.shape[1], len(classes)), classes
        return flatten_sklearn(est, X.shape[1], 1), None
    except Exception as e:  # noqa: BLE001
        _logger.warning("Failed to build a stat model because: {}".format(e))
        return None, None
