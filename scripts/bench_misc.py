"""delphi.misc on the C4-shaped table (100M x 32 dictionary codes, resident in HBM): device time of
describe (dr_scan_hist), toErrorMap (dr_error_map), injectNull (dr_null_bits) and splitInputTable (k = 8,
both algorithms: dr_kmeans_assign + dr_cooc per iteration, plus the host's P tables and centre updates),
each kernel's achieved bytes/s against its algorithmic bytes, and one sampled check of the final
assignment against the oracle's explicit row vectors.  Prints one JSON object; needs a CUDA device.

    python scripts/bench_misc.py [--rows 100000000] [--cols 32] [--k 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-data-repair-plugin_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def timed(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--cols", type=int, default=32)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample", type=int, default=20_000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_misc.py needs a CUDA device")
    from oracle import misc as OM
    from repair import cluster
    from repair._native import Context, profile_summary
    from repair.synth import SynthSpec, generate_torch
    dev = torch.device("cuda", 0)
    ctx = Context.acquire(0)
    n, K = args.rows, args.cols
    spec = SynthSpec.c4(n_rows=n, n_cols=K)
    codes = generate_torch(spec, dev)
    cols = [codes[i] for i in range(K)]
    dom = spec.dom
    torch.cuda.synchronize()
    res = {"card": card(), "rows": n, "cols": K, "k": args.k}

    # describe: one dr_scan_hist pass (4 B per cell in)
    off = np.concatenate([[0], np.cumsum([d + 1 for d in dom])]).astype(np.int64)
    hist = torch.zeros(int(off[-1]), dtype=torch.int64, device=dev)
    t = timed(torch, lambda: (hist.zero_(), ctx.scan_hist(cols, dom, n, [None] * K, hist)), args.reps)
    res["describe_scan_hist"] = {"s": t, "bytes": 4 * n * K, "GBps": 4 * n * K / t / 1e9}
    h = hist.cpu().numpy()
    hists = [h[off[i]:off[i + 1]] for i in range(K)]

    # toErrorMap: 4 attributes with errors (n / 8 B of bitmap each in), n K characters out
    words = (n + 31) // 32
    maps = [None] * K
    for i in (1, 5, 9, 20):
        if i < K:
            maps[i] = torch.randint(-2 ** 31, 2 ** 31 - 1, (words,), dtype=torch.int32, device=dev)
    out = torch.empty(n * K, dtype=torch.uint8, device=dev)
    t = timed(torch, lambda: ctx.error_map(maps, n, out), args.reps)
    b = n * K + sum(words * 4 for m in maps if m is not None)
    res["toErrorMap_error_map"] = {"s": t, "bytes": b, "GBps": b / t / 1e9}
    del out, maps

    # injectNull on every column: validity bits (dr_valid_bits, not timed) -> dr_null_bits, n / 8 B in + out each
    valid = [torch.zeros(words, dtype=torch.int32, device=dev) for _ in range(K)]
    for i in range(K):
        ctx.valid_bits(cols[i], n, valid[i])
    kept = [torch.empty(words, dtype=torch.int32, device=dev) for _ in range(K)]
    t = timed(torch, lambda: [ctx.null_bits(valid[i], 0, n, 0, 12345 + i, 0.01, kept[i]) for i in range(K)],
              args.reps)
    b = 2 * 4 * words * K
    res["injectNull_null_bits"] = {"s": t, "bytes": b, "GBps": b / t / 1e9}
    del valid, kept

    # splitInputTable, both algorithms
    strings = [["v%03d" % v for v in range(d)] for d in dom]
    feats = cluster.QgramFeatures(strings, hists, 2)
    res["vocabulary_terms"] = feats.n_terms
    res["P_bytes_kmeans"] = int((sum(d + 1 for d in dom) * args.k + args.k) * 8)
    for alg in ("bisect-kmeans", "kmeans++"):
        dk = cluster.DeviceKMeans(ctx, cols, feats, n, dev)
        info = {}
        torch.cuda.synchronize()
        ctx.profile = []
        t0 = time.perf_counter()
        if alg == "bisect-kmeans":           # the reference's crossed names: k-means
            cluster.kmeans(dk, args.k, info)
        else:
            cluster.bisecting_kmeans(dk, args.k, hists, n, info)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        prof = profile_summary(ctx)
        ctx.profile = None
        n_assign, t_assign = prof.get("kmeans_assign", (0, 0.0))
        n_cooc, t_cooc = prof.get("cooc", (0, 0.0))
        t_assign, t_cooc = t_assign / 1e3, t_cooc / 1e3
        a_bytes = (4 * K + 4) * n if alg == "bisect-kmeans" else (4 * K + 8) * n
        c_bytes = 4 * (K + 1) * n
        r = {"wall_s": wall, "assign_calls": n_assign, "cooc_calls": n_cooc,
             "assign_s_per_call": t_assign / max(n_assign, 1), "cooc_s_per_call": t_cooc / max(n_cooc, 1),
             "host_s": dk.host_s, "other_s": wall - t_assign - t_cooc - dk.host_s,
             "assign_GBps": a_bytes * n_assign / max(t_assign, 1e-12) / 1e9,
             "cooc_GBps": c_bytes * n_cooc / max(t_cooc, 1e-12) / 1e9,
             "assign_bytes_per_call": a_bytes, "cooc_bytes_per_call": c_bytes}
        if alg == "bisect-kmeans":
            r["iterations"] = info["iterations"]
            r["s_per_lloyd_iteration"] = wall / max(info["iterations"], 1)
            # one sampled check: the final assignment against the oracle's explicit row vectors
            rng = np.random.default_rng(1)
            rows = np.sort(rng.choice(n, size=args.sample, replace=False))
            idx = torch.from_numpy(rows).to(dev)
            sc = [c.index_select(0, idx).cpu().numpy() for c in cols]
            got = dk.labels.index_select(0, idx).cpu().numpy()
            P, mu_sq = feats.p_table(info["centres"])
            exact = OM.assign_from_p(sc, feats.dom, feats.p_off, P, mu_sq)
            import pandas as pd
            words_ = np.array(["v%03d" % i for i in range(64)] + [None], dtype=object)
            frame = pd.DataFrame({"c%02d" % i: words_[np.where(sc[i] < 0, 64, sc[i])] for i in range(K)})
            x, terms = OM.bags(frame, list(frame.columns), 2)
            pos = {g: i for i, g in enumerate(feats.terms)}
            cen = np.zeros((len(info["centres"]), len(terms)))
            for j, g in enumerate(terms):
                cen[:, j] = info["centres"][:, pos[g]]
            d = OM.sq_dist(x, cen)
            want = np.argmin(d, axis=1)
            diff = np.nonzero(got != want)[0]
            near = [int(i) for i in diff if abs(d[i, got[i]] - d[i, want[i]]) <= 1e-9 * max(d[i, want[i]], 1.0)]
            r["sample_check"] = {"rows": int(args.sample), "bit_identical_to_p_formula": bool(np.array_equal(got, exact)),
                                 "differ_from_row_vectors": int(len(diff)), "of_which_near_ties": len(near)}
        else:
            r["levels"] = info["levels"]
            r["leaves"] = info["n_leaves"]
        res["split_" + alg] = r
    Context.release(ctx)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
