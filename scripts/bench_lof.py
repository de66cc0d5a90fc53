"""LOFOutlierErrorDetector at scale: per-call CUDA-event times of the LOF path on a seeded 100M-row
continuous column at three distinct-value regimes, each with 1 % NULLs, next to a whole Engine.detect
pass with GaussianOutlierErrorDetector on the same column.

    python scripts/bench_lof.py [--rows 100000000] [--reps 5] [--samples 50000] [--out FILE]

Every timed run is verified: `--samples` entries are re-scored on the host by the oracle, each from its own
+-3k neighbourhood (oracle/lof.py: neighbourhoods / lof_at), and the flagged-row count is checked against
the verdicts and the global counts.  Prints one JSON line; nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "spark-data-repair-plugin_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
# dr_lof_score algorithmic bytes per entry: pass 1 reads u, cnt (16) and writes kdist (8); pass 2 reads u,
# cnt, kdist (24) and writes lrd (8); pass 3 reads u, cnt, lrd (24) and writes the verdict (1)
SCORE_BYTES_PER_ENTRY = 16 + 8 + 24 + 8 + 24 + 1
FLAG_BYTES_PER_ROW = 4      # one int32 code per row (the bitmap is 1 bit per row)


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = "unavailable ({})".format(type(e).__name__)
    return name, q


def make_column(torch, n, regime, seed, device):
    """Seeded float64 column on the device (NaN = NULL) -> (values, codes int32, host dictionary)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    v = torch.randn(n, generator=g, dtype=torch.float64, device=device)
    if regime == "d100":
        v = torch.round(v * 12.0)                       # ~100 distinct values
    elif regime == "d1e6":
        v = torch.round(v * 1.0e5) / 1.0e5              # ~1e6 distinct values
    null = torch.rand(n, generator=g, device=device) < 0.01
    v[null] = float("nan")
    valid = ~null
    uniq, inv = torch.unique(v[valid], sorted=True, return_inverse=True)
    codes = torch.full((n,), -1, dtype=torch.int32, device=device)
    codes[valid] = inv.to(torch.int32)
    del inv
    return v, codes, uniq.cpu().numpy()


def build_engine(torch, v, codes, dictionary, ctx):
    from repair.engine import Engine
    from repair.table import ROW_ALIGN, Column, DeviceTable, EncodedTable
    n = int(v.numel())
    n_pad = (n + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN
    c = torch.full((1, n_pad), -1, dtype=torch.int32, device=v.device)
    c[0, :n] = codes
    vals = torch.full((1, n_pad), float("nan"), dtype=torch.float64, device=v.device)
    vals[0, :n] = v
    col = Column("v", "float", dictionary, lambda: c[0, :n].cpu().numpy(), None)
    t = EncodedTable("tid", lambda: np.arange(n, dtype=np.int64), "int", [col], n_rows=n)
    dt = DeviceTable(t, v.device, codes=c, values=vals)
    return Engine(t, 0, device_table=dt, ctx=ctx)


def timed(torch, fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    e.synchronize()
    return out, s.elapsed_time(e) / 1e3


def run_regime(torch, regime, args, ctx):
    from oracle import lof as OL
    from repair.errors import ErrorModelOptions
    dev = torch.device("cuda", 0)
    v, codes, dictionary = make_column(torch, args.rows, regime, args.seed, dev)
    engine = build_engine(torch, v, codes, dictionary, ctx)
    del v, codes
    u = np.asarray(dictionary, dtype=np.float64)
    times = {k: [] for k in ("count_hist", "median", "entries", "lof_score", "lof_flag", "detect_lof",
                             "detect_gaussian")}
    opts = ErrorModelOptions.resolve({})
    checked = None
    for rep in range(args.reps + 1):          # rep 0 warms every shape up
        hist, t_h = timed(torch, lambda: engine.raw_value_counts_dev("v"))
        (_, _), t_m = timed(torch, lambda: engine.lof_median(u, hist))
        (d_u, cnt, k, entry, inserted), t_e = timed(torch, lambda: engine.lof_entries(u, hist))
        n_e = int(d_u.numel())
        verdict = torch.empty(n_e, dtype=torch.uint8, device=dev)
        kdist = torch.empty(n_e, dtype=torch.float64, device=dev)
        lrd = torch.empty(n_e, dtype=torch.float64, device=dev)
        lof = torch.empty(n_e, dtype=torch.float64, device=dev)
        _, t_s = timed(torch, lambda: ctx.lof_score(d_u, cnt, k, verdict, kdist, lrd, lof))
        null_verdict = bool(verdict[entry].item()) if entry >= 0 else False
        lut = torch.cat([verdict[:entry], verdict[entry + 1:]]) if inserted else verdict
        bm = engine.new_bitmap()
        _, t_f = timed(torch, lambda: ctx.lof_flag(engine.dt.col("v"), engine.n_rows, lut, len(u), null_verdict, bm))
        if rep == 0:
            checked = verify(torch, OL, engine, args, d_u, cnt, k, verdict, kdist, lrd, lof, bm, entry, inserted, hist)
        del kdist, lrd, lof
        _, t_dl = timed(torch, lambda: engine.detect([{"type": "lof"}], None, 80, opts))
        engine.reset()
        _, t_dg = timed(torch, lambda: engine.detect([{"type": "outlier"}], None, 80, opts))
        engine.reset()
        if rep == 0:
            continue
        for key, t in zip(times, (t_h, t_m, t_e, t_s, t_f, t_dl, t_dg)):
            times[key].append(t)
    med = {k: float(np.median(t)) for k, t in times.items()}
    out = {"regime": regime, "rows": args.rows, "distinct": len(u), "entries": n_e, "k": k,
           "median_inserted": bool(inserted), "times_s": med,
           "lof_score_GBps": SCORE_BYTES_PER_ENTRY * n_e / med["lof_score"] / 1e9,
           "lof_score_bytes_per_entry": SCORE_BYTES_PER_ENTRY,
           "lof_flag_GBps": FLAG_BYTES_PER_ROW * args.rows / med["lof_flag"] / 1e9,
           "lof_score_share_of_hbm_peak": SCORE_BYTES_PER_ENTRY * n_e / med["lof_score"] / HBM_BYTES_PER_S,
           "lof_flag_share_of_hbm_peak": FLAG_BYTES_PER_ROW * args.rows / med["lof_flag"] / HBM_BYTES_PER_S}
    out.update(checked)
    return out


def verify(torch, OL, engine, args, d_u, cnt, k, verdict, kdist, lrd, lof, bm, entry, inserted, hist):
    """Sampled entries re-scored by the oracle (bit for bit) + the flagged-row count from the verdicts."""
    n_e = int(d_u.numel())
    rng = np.random.default_rng(args.seed + 1)
    idx = np.unique(np.r_[rng.choice(n_e, size=min(args.samples, n_e), replace=False), 0, n_e - 1])
    flat, s_lo, s_hi, centre = OL.neighbourhoods(n_e, k, idx)
    ti = torch.from_numpy(flat).to(d_u.device)
    want = OL.lof_at(d_u[ti].cpu().numpy(), cnt[ti].cpu().numpy(), s_lo, s_hi, k, centre)
    ts = torch.from_numpy(idx).to(d_u.device)
    got = [t[ts].cpu().numpy() for t in (kdist, lrd, lof)] + [verdict[ts].cpu().numpy().astype(bool)]
    bad = np.zeros(len(idx), dtype=bool)
    for g, w in zip(got, want):
        bad |= g != w
    mism = int(bad.sum())
    # cells: rows of flagged entries (global counts, NULL rows through the median's entry) == bitmap popcount
    c_rows = hist[1:]
    v_codes = torch.cat([verdict[:entry], verdict[entry + 1:]]) if inserted else verdict
    expect = int((c_rows * v_codes.to(torch.int64)).sum().item())
    if entry >= 0:
        expect += int(hist[0].item()) * int(verdict[entry].item())
    cells = engine.ctx.bitmap_count(bm, engine.n_rows)
    return {"verify_sampled_entries": len(idx), "verify_mismatches": mism, "flagged_cells": cells,
            "flagged_cells_expected": expect, "cell_count_ok": cells == expect}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--regimes", default="d100,d1e6,all")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=50_000)
    ap.add_argument("--seed", type=int, default=20260)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_lof.py needs a CUDA device")
    from repair._native import Context
    name, power = gpu_info()
    ctx = Context.acquire(0)
    t0 = time.time()
    results = []
    for regime in args.regimes.split(","):
        results.append(run_regime(torch, regime, args, ctx))
        print(json.dumps(results[-1]), file=sys.stderr, flush=True)   # progress, one regime per line
        torch.cuda.empty_cache()
    line = {"gpu": name, "power_limit_and_max_sm_clock": power, "results": results,
            "total_mismatches": sum(r["verify_mismatches"] for r in results),
            "all_cell_counts_ok": all(r["cell_count_ok"] for r in results), "wall_s": time.time() - t0}
    Context.release(ctx)
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
