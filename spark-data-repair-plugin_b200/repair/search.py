"""Hyper-parameter search of the repair-model producer.

The reference tunes seven LightGBM parameters per model with hyperopt's TPE under k-fold cross
validation (``train.py:133-229``: ``fmin(tpe.suggest, max_evals, early_stop_fn=no_progress_loss /
timeout)``, ``StratifiedKFold`` / ``KFold(n_splits, shuffle=True)``, scorer ``f1_macro`` /
``neg_mean_squared_error``).  hyperopt is not available offline, so the search PATH is unpinned (and
unseeded CV shuffles make it non-deterministic upstream anyway); what is reproduced is the search
SPACE, the objective, the budget / early-stop options and the TPE recipe: random start-up trials,
then candidates drawn from a Parzen estimator of the good trials and ranked by l(x) / g(x).

Deviations, all deterministic: trial 0 evaluates LightGBM's defaults (hyperopt's first trial is a
random draw), so ``model.hp.max_evals=1`` -- what the reference's own unit tests use -- trains the
default model without any cross-validation; CV shuffles and the sampler are seeded (42).
"""
import logging
import math
import time

import numpy as np

_logger = logging.getLogger("repair")

# (name, kind, low, high): hp.quniform(q=1) / hp.uniform / hp.loguniform (bounds in log space)  train.py:148-156
SPACE = [
    ("num_leaves", "quniform", 2.0, 100.0),
    ("subsample", "uniform", 0.5, 1.0),
    ("subsample_freq", "quniform", 1.0, 20.0),
    ("colsample_bytree", "uniform", 0.01, 1.0),
    ("min_child_samples", "quniform", 1.0, 50.0),
    ("min_child_weight", "loguniform", -3.0, 1.0),
    ("reg_lambda", "loguniform", -2.0, 3.0),
]
# LightGBM 3.3.1 defaults of the tuned parameters (the model the fixed parameters alone give)
DEFAULTS = {"num_leaves": 31, "subsample": 1.0, "subsample_freq": 0, "colsample_bytree": 1.0,
            "min_child_samples": 20, "min_child_weight": 1e-3, "reg_lambda": 0.0}
INT_PARAMS = ("num_leaves", "subsample_freq", "min_child_samples")   # train.py:124-127

N_STARTUP, GAMMA, N_CANDIDATES = 20, 0.25, 24     # hyperopt.tpe defaults


def _to_params(vec):
    out = {}
    for (name, kind, _, _), v in zip(SPACE, vec):
        v = math.exp(v) if kind == "loguniform" else v
        out[name] = int(round(v)) if name in INT_PARAMS else float(v)
    return out


def _draw_prior(rng):
    vec = []
    for _, kind, lo, hi in SPACE:
        v = rng.uniform(lo, hi)
        vec.append(float(np.clip(np.round(v), lo, hi)) if kind == "quniform" else float(v))
    return vec


def _parzen(obs, lo, hi):
    """Adaptive Parzen estimator of hyperopt.tpe: one Gaussian per observation plus the prior in the
    middle of the range; a component's width is its distance to the farther neighbour, clipped."""
    prior_mu, prior_sigma = 0.5 * (lo + hi), hi - lo
    mus = np.sort(np.asarray(list(obs) + [prior_mu], dtype=np.float64))
    if len(mus) == 1:
        sig = np.array([prior_sigma])
    else:
        gaps = np.diff(mus)
        sig = np.maximum(np.r_[gaps[0], gaps], np.r_[gaps, gaps[-1]])
    sig = np.clip(sig, prior_sigma / min(100.0, 1.0 + len(mus)), prior_sigma)
    sig[np.argmin(np.abs(mus - prior_mu))] = prior_sigma
    return mus, sig


def _log_pdf(x, mus, sig, lo, hi):
    z = (x[:, None] - mus[None, :]) / sig[None, :]
    comp = -0.5 * z * z - np.log(sig[None, :] * math.sqrt(2.0 * math.pi))
    # truncation to [lo, hi]
    cdf = lambda t: 0.5 * (1.0 + np.vectorize(math.erf)((t - mus) / (sig * math.sqrt(2.0))))  # noqa: E731
    mass = np.maximum(cdf(hi) - cdf(lo), 1e-12)
    comp = comp - np.log(mass)[None, :]
    m = comp.max(axis=1, keepdims=True)
    return (m[:, 0] + np.log(np.exp(comp - m).sum(axis=1))) - math.log(len(mus))


def _suggest(rng, trials):
    """One TPE proposal from [(vector, loss)]: per dimension, candidates from l(x) (good trials), the
    one with the largest l(x) / g(x) wins (dimensions are independent, as in hyperopt)."""
    losses = np.asarray([t[1] for t in trials])
    order = np.argsort(losses, kind="stable")
    n_below = min(int(math.ceil(GAMMA * math.sqrt(len(trials)))), 25)
    below, above = order[:n_below], order[n_below:]
    vec = []
    for d, (_, kind, lo, hi) in enumerate(SPACE):
        good = [trials[i][0][d] for i in below]
        bad = [trials[i][0][d] for i in above]
        mg, sg = _parzen(good, lo, hi)
        mb, sb = _parzen(bad, lo, hi)
        comp = rng.integers(0, len(mg), size=N_CANDIDATES)
        cand = np.clip(rng.normal(mg[comp], sg[comp]), lo, hi)
        if kind == "quniform":
            cand = np.clip(np.round(cand), lo, hi)
        score = _log_pdf(cand, mg, sg, lo, hi) - _log_pdf(cand, mb, sb, lo, hi)
        vec.append(float(cand[int(np.argmax(score))]))
    return vec


def cv_folds(y, is_discrete, n_splits, seed=42):
    """StratifiedKFold / KFold(n_splits, shuffle=True) (train.py:158-161), seeded."""
    from sklearn.model_selection import KFold, StratifiedKFold
    import warnings
    n = len(y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)   # classes with fewer members than folds (train.py:143-145)
        if is_discrete:
            return list(StratifiedKFold(n_splits=n_splits, shuffle=True, random_state=seed).split(np.zeros(n), y))
        return list(KFold(n_splits=n_splits, shuffle=True, random_state=seed).split(np.zeros(n)))


def score(y_true, y_pred, is_discrete):
    """f1_macro / neg_mean_squared_error (train.py:157)."""
    if is_discrete:
        from sklearn.metrics import f1_score
        return float(f1_score(y_true, y_pred, average="macro"))
    d = np.asarray(y_true, dtype=np.float64) - np.asarray(y_pred, dtype=np.float64)
    return -float(np.mean(d * d))


# trial 0 under boosting_type rf: LightGBM refuses rf without row bagging or feature sub-sampling, so the
# defaults draw a new bag per tree at the bootstrap's expected share of distinct rows
RF_DEFAULTS = dict(DEFAULTS, subsample=0.632, subsample_freq=1)


def search(evaluate, max_evals, no_progress_loss, timeout, seed=42, defaults=None):
    """``fmin`` of train.py:198-209.  evaluate(params) -> loss (= -mean CV score; exceptions count as
    0.0 like train.py:176-180), or (loss, per-fold losses).  -> (best params, best loss, number of
    evaluations).  defaults: trial 0 and the ``max_evals <= 1`` result (LightGBM's ``DEFAULTS`` if None).

    One deliberate deviation from hyperopt's plain argmin: k-fold CV on a few hundred rows is noisy, so a
    tuned configuration only replaces LightGBM's defaults (trial 0) when it beats them by more than one
    standard error of the defaults' own fold losses (the "one-standard-error rule" of model selection).
    Without it a short search degrades heavy-tailed regression targets (boston CRIM: 8 % better CV MSE,
    12 % worse RMSE on the repaired cells) while helping others (TAX: 23 % better CV MSE, 24 % better RMSE)."""
    defaults = DEFAULTS if defaults is None else defaults
    if max_evals <= 1:
        return dict(defaults), None, 0
    rng = np.random.default_rng(seed)
    trials = []          # (vector in search space, loss)
    best_loss, best_params, since_best = None, dict(defaults), 0
    default_loss, default_se = None, 0.0
    t0 = time.time()
    for it in range(int(min(max_evals, 1 << 30))):
        if it == 0:
            params, vec = dict(defaults), None
        else:
            vec = _draw_prior(rng) if len(trials) < N_STARTUP else _suggest(rng, trials)
            params = _to_params(vec)
        folds = None
        try:
            got = evaluate(params)
            if isinstance(got, tuple):
                got, folds = got
            loss = float(got)
        except Exception as e:  # noqa: BLE001  (train.py:176-180: e.g. previously unseen labels in a fold)
            _logger.warning("{}: {}".format(e.__class__, e))
            loss = 0.0
        if it == 0:
            default_loss = loss
            if folds is not None and len(folds) > 1:
                default_se = float(np.std(np.asarray(folds, dtype=np.float64), ddof=1) / math.sqrt(len(folds)))
        if vec is not None:
            trials.append((vec, loss))
        if best_loss is None or loss < best_loss:
            best_loss, best_params, since_best = loss, params, 0
        else:
            since_best += 1
        if since_best >= no_progress_loss or (timeout > 0 and time.time() - t0 > timeout):
            break
    if default_loss is not None and best_loss is not None and not best_loss < default_loss - default_se:
        best_params, best_loss = dict(defaults), default_loss     # not a significant improvement
    _logger.info("hyperopt: #eval={}/{}".format(it + 1, max_evals))
    return best_params, best_loss, it + 1
