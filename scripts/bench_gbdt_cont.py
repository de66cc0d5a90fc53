"""Times the GPU trainer against scikit-learn's histogram GBDT on continuous features, and boston end to end.

Models with a continuous target or feature train on the GPU when model.lgb.boosting_type, reg_alpha or
min_split_gain is set, and on scikit-learn otherwise.  This measures both on the same problems:

* verify: before timing, one reduced configuration per boosting type (900 rows, 9 rounds) on quantile-
  binned continuous columns is checked bit for bit against oracle/gbdt_boost.py;
* trainer: gbdt.train_gpu (bins included) against train.build_model without search, both 300 rounds at
  learning rate 0.01, depth 7, on a seeded 10 000-row problem with 13 continuous features (NULLs, a
  duplicate-heavy column, a > 254-value column) and a regression, a binary and an 8-class target; wall
  time around a device synchronise, median of --reps after one warm-up;
* held-out MSE of the regression target, both trainers trained on the same 80 % and scored on the rest;
* boston: RepairModel.run() on tests/golden/bin_boston.csv with the NULL detector, training included,
  at model.hp.max_evals=1 and 3, under goss (GPU trainer) and at the defaults (scikit-learn).

Prints one JSON line with the card name, power limit and max SM clock; nothing is written to the tree.
"""
import argparse
import json
import logging
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "spark-data-repair-plugin_b200"), os.path.join(ROOT, "scripts")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_gbdt import card  # noqa: E402

MODES = {"gbdt": {}, "goss": {"boosting": "goss"}, "dart": {"boosting": "dart"},
         "rf": {"boosting": "rf", "subsample": 0.632, "subsample_freq": 1}}


def cont_problem(n, seed=7):
    """13 float64 columns: NULLs in several, one duplicate-heavy, one with thousands of values ->
    (X [n, 13], regression target, signal)."""
    rng = np.random.default_rng(seed)
    X = np.round(rng.normal(size=(n, 13)) * [1, 2, 5, 0.5, 10, 1, 3, 1, 1, 2, 7, 1, 100], 2)
    X[:, 2] = rng.choice([0.0, 1.5, 2.25, 9.0, 30.0], size=n)             # duplicate-heavy
    X[:, 12] = np.round(rng.normal(size=n) * 300.0, 3)                     # > 254 distinct values
    for j in (0, 4, 7, 12):
        X[rng.random(n) < 0.08, j] = np.nan
    sig = np.nan_to_num(X[:, 0]) * 1.5 + (X[:, 2] > 2) * 3.0 + np.nan_to_num(X[:, 4]) * 0.2 + \
        np.sin(np.nan_to_num(X[:, 12]) / 150.0) * 2.0 + X[:, 1] * X[:, 3]
    return X, sig + rng.normal(size=n) * 0.5, sig


def binned(X, max_bin=255):
    from repair import gbdt as G
    cols = {str(j): X[:, j] for j in range(X.shape[1])}
    return G.bin_sample([{"attr": a, "type": "cont"} for a in cols], {}, {}, max_bin=max_bin, sample_values=cols)


def targets(y_reg, sig, rng):
    q = np.quantile(sig, np.linspace(0, 1, 9)[1:-1])
    return {"regression": (y_reg, 1), "binary": ((sig + rng.normal(size=len(sig)) > np.median(sig)).astype(np.int64), 2),
            "8-class": (np.searchsorted(q, sig + rng.normal(size=len(sig)) * 0.5).astype(np.int64), 8)}


def verify(ctx, torch):
    """-> {mode: [mismatching arrays]} of the reduced configurations against the oracle."""
    from oracle import gbdt_boost as OB
    from repair import gbdt as G
    X, y_reg, sig = cont_problem(900, 3)
    bins, n_bins, values = binned(X)
    idx = [np.arange(256, dtype=np.float64)] * len(n_bins)
    hi_lo = [(v, v) if np.ndim(v) == 1 else (v[0], v[1]) for v in values]
    out = {}
    for name, (y, C) in targets(y_reg, sig, np.random.default_rng(1)).items():
        w = G.class_weights(y, C, True) if C > 1 else None
        for mode, kw in MODES.items():
            kw = dict(kw, num_leaves=15, min_data_in_leaf=10, reg_alpha=0.3, min_split_gain=0.01)
            k, yk, kwk = 0, y, kw
            if C == 1:                        # the oracle on the target as train_gpu scales it, scaled back
                gs = OB.goss_counts(len(y))[3] if mode == "goss" else 0
                k = G.regression_scale(y, G.initial_scores(y, 1, None)[0], len(y), gs)
                yk = np.ldexp(y, -k)
                kwk = dict(kw, reg_alpha=float(np.ldexp(kw["reg_alpha"], -k)),
                           min_split_gain=float(np.ldexp(kw["min_split_gain"], -2 * k)))
            want = OB.to_flat_forest(OB.train(bins, n_bins, yk, C, w, 9, 0.25, 5, **kwk), idx, len(n_bins))
            want["baseline"], want["value"] = np.ldexp(want["baseline"], k), np.ldexp(want["value"], k)
            # plain midpoints: the problem's values are finite and rounded, so flatten's fallback never applies
            inner = np.asarray(want["feature"]) >= 0
            want["threshold"][inner] = [(hi_lo[f][0][b] + hi_lo[f][1][b + 1]) / 2.0 for f, b in
                                        zip(np.asarray(want["feature"])[inner], want["threshold"][inner].astype(int))]
            got = G.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, values, y, C,
                              w if w is not None else np.ones(len(y)), 9, 0.25, 5, **kw)
            out["{}/{}".format(name, mode)] = [k for k in want if not np.array_equal(np.asarray(got[k]),
                                                                                      np.asarray(want[k]))]
    return out


def _median_time(fn, reps, sync):
    fn()
    sync()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = fn()
        sync()
        times.append(time.perf_counter() - t0)
    return round(statistics.median(times), 4), res


def trainers(ctx, torch, rows, reps):
    from oracle.forest import forest_predict
    from repair import gbdt as G
    from repair.train import build_model
    X, y_reg, sig = cont_problem(rows)
    opts = {"model.hp.max_evals": "1"}            # 300 rounds, learning rate 0.01, depth 7: the defaults
    results, mse = [], {}
    for name, (y, C) in targets(y_reg, sig, np.random.default_rng(2)).items():
        w = G.class_weights(y, C, True) if C > 1 else np.ones(len(y))

        def gpu(kw):
            b = binned(X)
            return G.train_gpu(ctx, torch.device("cuda", 0), b[0], b[1], b[2], y, C, w, 300, 0.01, 7, **kw)
        for mode, kw in MODES.items():
            t, _ = _median_time(lambda: gpu(kw), reps, torch.cuda.synchronize)
            results.append({"target": name, "trainer": "gpu", "mode": mode, "wall_s": t})
        t, _ = _median_time(lambda: build_model(X, y, C > 1, C if C > 1 else 0, opts), reps, lambda: None)
        results.append({"target": name, "trainer": "sklearn", "mode": "gbdt", "wall_s": t})
        print(json.dumps(results[-1]), file=sys.stderr, flush=True)
    # held-out MSE of the regression target: the same 80 / 20 split for both trainers
    perm = np.random.default_rng(5).permutation(rows)
    tr, te = perm[: rows * 4 // 5], perm[rows * 4 // 5:]
    b = binned(X[tr])
    for mode, kw in MODES.items():
        f = G.train_gpu(ctx, torch.device("cuda", 0), b[0], b[1], b[2], y_reg[tr], 1, np.ones(len(tr)), 300, 0.01, 7,
                        **kw)
        mse["gpu_" + mode] = round(float(np.mean((forest_predict(f, X[te]) - y_reg[te]) ** 2)), 4)
    f, _ = build_model(X[tr], y_reg[tr], False, 0, opts)
    mse["sklearn_gbdt"] = round(float(np.mean((forest_predict(f, X[te]) - y_reg[te]) ** 2)), 4)
    mse["mean_fill"] = round(float(np.mean((y_reg[tr].mean() - y_reg[te]) ** 2)), 4)
    return results, mse


def boston(reps):
    import pandas as pd
    from repair import RepairModel
    from repair.errors import NullErrorDetector
    df = pd.read_csv(os.path.join(ROOT, "tests", "golden", "bin_boston.csv"))
    df["CHAS"] = df["CHAS"].map(lambda v: None if v != v else str(v))
    df["RAD"] = df["RAD"].map(lambda v: None if v != v else str(int(v)))
    out = []
    for evals in (1, 3):
        for mode in ("gbdt", "goss"):
            def run():
                rm = RepairModel().setInput(df).setRowId("tid").setErrorDetectors([NullErrorDetector()])
                rm.option("model.hp.max_evals", str(evals)).option("model.lgb.boosting_type", mode)
                rm.run()
                return rm
            t, rm = _median_time(run, reps, lambda: None)
            out.append({"max_evals": evals, "boosting_type": mode, "trainer": "gpu" if mode != "gbdt" else "sklearn",
                        "wall_s": t, "training_s": round(rm.last_run["elapsed_training"], 3)
                        if "elapsed_training" in rm.last_run else None})
            print(json.dumps(out[-1]), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--run-reps", type=int, default=1, help="timed boston runs per configuration")
    args = ap.parse_args()
    logging.getLogger("repair").setLevel(logging.ERROR)
    import torch
    from repair._native import Context
    name, power = card()
    ctx = Context.acquire(0)
    t0 = time.time()
    mismatches = verify(ctx, torch)
    ok = not any(mismatches.values())
    print(json.dumps({"verify_ok": ok, "verify": mismatches}), file=sys.stderr, flush=True)
    results, mse = trainers(ctx, torch, args.rows, args.reps)
    Context.release(ctx)
    runs = boston(args.run_reps)
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "rows": args.rows, "rounds": 300,
                      "verify_ok": ok, "verify_mismatches": {k: v for k, v in mismatches.items() if v},
                      "trainer": results, "held_out_mse": mse, "boston_run": runs,
                      "wall_s": round(time.time() - t0, 1)}))


if __name__ == "__main__":
    main()
