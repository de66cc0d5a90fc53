"""Times the GPU trainer under each model.lgb.boosting_type (gbdt, goss, dart, rf) on C4-shaped models.

A C4 repair model: 10 000 training rows, 31 byte features with the domain sizes of repair/synth.py's C4
table, 300 rounds at learning rate 0.01, depth 7; a binary, an 8-class and a 64-class target.  rf runs
with subsample 0.632 every iteration (what the search's trial 0 uses under rf).  Per model: wall time
around a device synchronise (median of --reps after one warm-up) and kernel launches.

Before timing, one reduced configuration per mode (a few hundred rows, 20 rounds, learning rate 0.25 so
that goss samples from iteration 4 on) is checked bit for bit against oracle/gbdt_boost.py.  Prints one
JSON line with the card name, power limit and max SM clock; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "spark-data-repair-plugin_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

MODES = {"gbdt": {}, "goss": {"boosting": "goss"}, "dart": {"boosting": "dart"},
         "rf": {"boosting": "rf", "subsample": 0.632, "subsample_freq": 1}}


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = "unavailable ({})".format(type(e).__name__)
    return torch.cuda.get_device_name(0), q


def c4_problem(n, n_classes, seed):
    """bins of 31 features with C4's domain sizes (+ a missing bin), a target that depends on a few of them."""
    from repair import gbdt as G
    from repair.synth import domain_size
    rng = np.random.default_rng(seed)
    doms = [domain_size(i) for i in range(31)]
    bins = np.stack([rng.integers(0, d + 1, size=n) for d in doms], axis=1).astype(np.uint8)
    sig = bins[:, 3].astype(np.int64) * 5 + bins[:, 5] * 3 + bins[:, 12] + rng.integers(0, 4, size=n)
    y = (sig % n_classes).astype(np.int64)
    vals = [np.arange(d, dtype=np.float64) for d in doms]
    return bins, np.array([d + 1 for d in doms], dtype=np.int32), vals, y, G.class_weights(y, n_classes, True)


def verify(ctx, torch):
    """-> {mode: mismatching arrays} of the reduced configuration against the oracle."""
    from oracle import gbdt_boost as OB
    from repair import gbdt as G
    bins, n_bins, vals, y, w = c4_problem(400, 8, 11)
    out = {}
    for mode, kw in MODES.items():
        kw = dict(kw, num_leaves=15, min_data_in_leaf=10)
        if mode == "dart":
            kw.update(drop_rate=0.3, skip_drop=0.2)
        want = OB.to_flat_forest(OB.train(bins, n_bins, y, 8, w, 20, 0.25, 5, **kw), vals, bins.shape[1])
        got = G.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, vals, y, 8, w, 20, 0.25, 5, **kw)
        out[mode] = [k for k in want if not np.array_equal(np.asarray(got[k]), np.asarray(want[k]))]
    return out


def time_model(ctx, torch, bins, n_bins, vals, y, w, n_classes, kw, reps):
    from repair import gbdt as G
    run = lambda: G.train_gpu(ctx, torch.device("cuda", 0), bins, n_bins, vals, y, n_classes, w, 300, 0.01, 7,  # noqa
                              **kw)
    run()
    torch.cuda.synchronize()
    times, launches = [], 0
    for _ in range(reps):
        l0 = ctx.launch_count
        t0 = time.perf_counter()
        forest = run()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        launches = ctx.launch_count - l0
    return {"wall_s": round(statistics.median(times), 4), "launches": launches,
            "splits": int((np.asarray(forest["feature"]) >= 0).sum())}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=10_000)
    ap.add_argument("--classes", default="2,8,64")
    ap.add_argument("--modes", default="gbdt,goss,dart,rf")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from repair._native import Context
    name, power = card()
    ctx = Context.acquire(0)
    t0 = time.time()
    mismatches = verify(ctx, torch)
    print(json.dumps({"verify": mismatches}), file=sys.stderr, flush=True)
    results = []
    for c in [int(v) for v in args.classes.split(",")]:
        bins, n_bins, vals, y, w = c4_problem(args.rows, c, c)
        for mode in args.modes.split(","):
            r = dict(time_model(ctx, torch, bins, n_bins, vals, y, w, c, MODES[mode], args.reps), classes=c, mode=mode)
            results.append(r)
            print(json.dumps(r), file=sys.stderr, flush=True)   # progress, one model per line
    Context.release(ctx)
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "rows": args.rows, "rounds": 300,
                      "verify_mismatches": mismatches, "verify_ok": not any(mismatches.values()),
                      "results": results, "wall_s": round(time.time() - t0, 1)}))


if __name__ == "__main__":
    main()
