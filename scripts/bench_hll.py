"""Spark-compatible distinct counts at scale: dr_hll_dict over seeded high-cardinality string dictionaries, and
the time the opt-in mode adds to a C4-shaped detection pass.

    python scripts/bench_hll.py [--entries 1000000,100000000] [--rows 10000000] [--cols 16] [--reps 5] [--out FILE]

* dict: the dictionary (random bytes, lengths 4 - 28, Arrow layout) is generated on the device; the kernel is
  timed with CUDA events and its rate reported over the dictionary's string bytes (the int64 offsets it also
  reads are reported beside it).  The 10^6-entry registers are checked against oracle/hll.py.
* pass: RepairModel.run(detect_errors_only=True) over a synthetic C4 table (NULL + FD detectors), mode off and
  on alternately; the difference is mostly the full-table pair presence of the scored pairs.
Prints one JSON line; nothing is written to the tree.
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


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = "unavailable ({})".format(type(e).__name__)
    return name, q


def bench_dict(torch, ctx, n, reps, seed):
    from repair import hll as RH
    from repair._native import DR_HLL_KIND
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    lens = torch.randint(4, 29, (n,), generator=g, device=dev, dtype=torch.int64)
    off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(lens, 0, out=off[1:])
    del lens
    n_bytes = int(off[-1].item())
    data = torch.randint(0, 256, (n_bytes + 8,), generator=g, device=dev, dtype=torch.uint8)
    regs = torch.zeros(RH.M, dtype=torch.int32, device=dev)
    times = []
    for rep in range(reps + 1):        # rep 0 warms up
        regs.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        ctx.hll_dict(DR_HLL_KIND["string"], data, off, n, regs)
        e.record()
        e.synchronize()
        if rep:
            times.append(s.elapsed_time(e) / 1e3)
    t = float(np.median(times))
    regs_h = regs.cpu().numpy().astype(np.uint8)
    out = {"entries": n, "string_bytes": n_bytes, "offset_bytes": 8 * (n + 1), "k_hll_dict_s": t,
           "string_GBps": n_bytes / t / 1e9, "string_and_offsets_GBps": (n_bytes + 8 * (n + 1)) / t / 1e9,
           "share_of_hbm_peak": (n_bytes + 8 * (n + 1)) / t / HBM_BYTES_PER_S,
           "estimate": RH.distinct_count(regs_h, n)[0]}
    if n <= 2_000_000:
        from oracle import hll as H
        raw, o = data.cpu().numpy().tobytes(), off.cpu().numpy()
        want = H.registers(H.hash_bytes_many([raw[o[i]:o[i + 1]] for i in range(n)]))
        out["registers_match_oracle"] = bool(np.array_equal(want, regs_h))
    del data, off
    torch.cuda.empty_cache()
    return out


def bench_pass(torch, rows, cols, reps, seed):
    from repair import RepairModel, synth
    from repair.table import EncodedTable
    import parity_utils as PU
    spec = synth.SynthSpec.c4(rows, cols, seed=seed)
    t = EncodedTable.from_codes("tid", synth.column_names(cols), synth.generate_numpy(spec), spec.dom)
    specs = [{"type": "null"}, {"type": "constraint", "constraints": synth.fd_constraints(cols)}]
    times = {False: [], True: []}
    outs = {}
    for rep in range(reps + 1):
        for mode in (False, True):
            rm = RepairModel().setEncodedInput(t).setErrorDetectors(PU.make_detectors(specs))
            rm.setSparkCompatibleDistinctCounts(mode)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = rm.run(detect_errors_only=True)
            torch.cuda.synchronize()
            if rep:
                times[mode].append(time.perf_counter() - t0)
            else:
                res = rm.last_run["detect"]
                outs[mode] = {"cells": len(out), "scored_pairs": len(rm.last_run.get("distinct_count_provenance", {})
                                                                      .get("pairs", {})),
                              "disc_attrs": len(res.disc_attrs)}
    off, on = float(np.median(times[False])), float(np.median(times[True]))
    return {"rows": rows, "cols": cols, "detect_off_s": off, "detect_on_s": on, "added_s": on - off,
            "runs_off_s": times[False], "runs_on_s": times[True], "off": outs[False], "on": outs[True]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--entries", default="1000000,100000000")
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--cols", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_hll.py needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from repair._native import Context
    name, power = gpu_info()
    ctx = Context.acquire(0)
    t0 = time.time()
    dicts = []
    for n in [int(v) for v in args.entries.split(",") if v]:
        dicts.append(bench_dict(torch, ctx, n, args.reps, args.seed))
        print(json.dumps(dicts[-1]), file=sys.stderr, flush=True)
    Context.release(ctx)
    pas = bench_pass(torch, args.rows, args.cols, args.reps, args.seed) if args.rows > 0 else None
    line = {"gpu": name, "power_limit_and_max_sm_clock": power, "dict": dicts, "pass": pas, "wall_s": time.time() - t0}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
