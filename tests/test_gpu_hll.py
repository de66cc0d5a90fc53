"""Spark-compatible HyperLogLog++ distinct counts on the device: dr_hll_dict / dr_hll_pairs registers
byte-identical to oracle/hll.py, and the opt-in mode through the public API (hospital's domain_stats equal
the values the reference pins, RepairSuite.scala:156-175, and the discretisation follows them)."""
import os
import socket

import numpy as np
import pandas as pd
import pytest

from conftest import GOLDEN
from oracle import hll as H
from test_hll_cpu import HOSPITAL_DOMAIN_STATS

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    from repair._native import Context
    c = Context.acquire(0)
    yield c
    Context.release(c)


def _device_regs(ctx, name, values, stype):
    from repair import hll as RH
    regs, hx = RH.column_registers(ctx, torch.device("cuda", 0), name, values, stype, hashes=True)
    return regs, hx[:len(values)].cpu().numpy().view(np.uint64)


def _strings():
    rng = np.random.default_rng(11)
    alphabet = list("abcxyz0129 _-") + ["é", "ß", "日", "本", "語", "😀"]
    out = [""]
    for n in range(1, 101):          # every XXH64 length path: 32-byte stripes, 8-, 4- and 1-byte tails
        for _ in range(3):
            out.append("".join(rng.choice(alphabet, size=n)))
    return sorted(set(out))


def test_dict_registers_strings(ctx):
    vals = _strings()
    regs, hx = _device_regs(ctx, "s", vals, "string")
    assert np.array_equal(hx, H.hash_values(vals, "string"))
    assert regs.tobytes() == H.column_registers(vals, "string").tobytes()


@pytest.mark.parametrize("stype,dtype", [("int", np.int32), ("long", np.int64), ("float", np.float32),
                                         ("double", np.float64), ("boolean", np.int32)])
def test_dict_registers_numeric(ctx, stype, dtype):
    rng = np.random.default_rng(2)
    if stype == "boolean":
        vals = np.array([0.0, 1.0])
    elif stype in ("int", "long"):
        lim = 2 ** 31 - 1 if stype == "int" else 2 ** 53
        vals = np.unique(np.r_[0, 1, -1, -lim, lim, rng.integers(-lim, lim, size=5000)]).astype(np.float64)
    else:
        vals = np.unique(np.r_[-0.0, 1.5, -2.25, np.inf, -np.inf, rng.normal(size=5000)].astype(dtype)
                         ).astype(np.float64)
        vals = np.r_[vals, -0.0]        # -0.0 hashes as 0.0
    regs, hx = _device_regs(ctx, "n", vals, stype)
    assert np.array_equal(hx, H.hash_values(vals.astype(dtype), stype))
    assert regs.tobytes() == H.column_registers(vals.astype(dtype), stype).tobytes()


def test_dict_registers_one_million_entries(ctx):
    vals = ["k%07d-%s" % (i, "x" * (i % 41)) for i in range(1_000_000)]
    regs, _ = _device_regs(ctx, "big", vals, "string")
    assert regs.tobytes() == H.column_registers(vals, "string").tobytes()


@pytest.mark.parametrize("y_type", ["string", "int"])
def test_pair_registers(ctx, y_type):
    from repair import hll as RH
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(4)
    xs = _strings()[:90]
    ys = _strings()[90:160] if y_type == "string" else np.arange(41).astype(np.float64)
    pairs, want = [], []
    bits_all, regs = [], torch.zeros((3, H.M), dtype=torch.int32, device=dev)
    _, hx_dev = RH.column_registers(ctx, dev, "x", xs, "string", hashes=True)
    kind, data, off, _ = RH.value_buffers("y", ys, y_type, dev)
    hx = np.r_[np.uint64(42), H.hash_values(xs, "string")]
    for q, density in enumerate((0.02, 0.3, 1.0)):
        present = rng.random((len(xs) + 1, len(ys) + 1)) < density
        present[0, 0] = True
        flat = np.zeros((present.size + 31) // 32 * 32, dtype=bool)
        flat[:present.size] = present.reshape(-1)
        words = torch.from_numpy(np.packbits(flat, bitorder="little").view(np.int32).copy()).to(dev)
        bits_all.append(words)
        pairs.append((hx_dev, kind, data, off, len(xs), len(ys), words, regs[q]))
        y_vals = ys if y_type == "string" else ys.astype(np.int32)
        want.append(H.pair_registers(hx, y_vals, y_type, present))
    ctx.hll_pairs(pairs)
    got = regs.cpu().numpy().astype(np.uint8)
    for q in range(3):
        assert got[q].tobytes() == want[q].tobytes(), q


def _hospital():
    return pd.read_csv(os.path.join(GOLDEN, "hospital.csv"), dtype=str).astype({"tid": int})


def _given(df):
    """Error cells: every NULL Score cell and six ZipCode cells, in both halves of the table (each shard of a
    two-rank run holds cells of both attributes)."""
    rows = sorted(df.loc[df["Score"].isna(), "tid"].tolist())
    zips = [0, 1, 2, 500, 501, 502]
    return pd.DataFrame({"tid": rows + zips, "attribute": ["Score"] * len(rows) + ["ZipCode"] * len(zips)})


def _model(df, spark_ndv, thres=80):
    from repair import RepairModel
    from repair.errors import NullErrorDetector
    rm = RepairModel().setInput(df).setRowId("tid").setErrorDetectors([NullErrorDetector()])
    rm.setDiscreteThreshold(thres).setSparkCompatibleDistinctCounts(spark_ndv)
    rm.option("model.hp.max_evals", "1")
    return rm


def test_hospital_domain_stats_through_the_api():
    rm = _model(_hospital(), True)
    rm.run(detect_errors_only=True)
    res = rm.last_run["detect"]
    assert res.domain_stats == HOSPITAL_DOMAIN_STATS
    prov = rm.last_run["distinct_count_provenance"]
    assert set(prov["columns"].values()) == {"estimate"}
    # the scored pairs (all of Score's, both kept string columns): estimate or exact fallback as the oracle decides
    df = _hospital()
    assert prov["pairs"]
    for (x, y), how in prov["pairs"].items():
        seen = set(zip(df[x].where(df[x].notna(), None), df[y].where(df[y].notna(), None)))
        hashes = [H.spark_hash(b, "string", H.spark_hash(a, "string")) for a, b in seen]
        assert H.distinct_count(H.registers(hashes), len(seen))[1] == how, (x, y)
    off = _model(_hospital(), False)
    off.run(detect_errors_only=True)
    assert off.last_run["detect"].domain_stats["Sample"] == 333
    assert "distinct_count_provenance" not in off.last_run


def test_threshold_70_keeps_zipcode_and_drops_score():
    df = _hospital()
    score_nulls = set(df.loc[df["Score"].isna(), "tid"].tolist())
    assert len(score_nulls) == 167
    for spark_ndv in (True, False):
        rm = _model(df, spark_ndv, thres=70)
        cells = rm.run(detect_errors_only=True)
        assert set(cells.loc[cells["attribute"] == "Score", "tid"].tolist()) == score_nulls
        res = rm.last_run["detect"]
        assert ("ZipCode" in res.disc_attrs) == spark_ndv and ("Score" in res.disc_attrs) != spark_ndv
        assert ("Score" in res.target_columns) != spark_ndv
    # repairs: the Score NULL cells plus a few ZipCode cells as given error cells -- only the discretised one of
    # the two is repaired
    for spark_ndv in (True, False):
        rm = _model(df, spark_ndv, thres=70).setErrorCells(_given(df))
        rm.option("model.lgb.n_estimators", "8")
        out = rm.run()
        repaired = set(out.loc[out["repaired"].notna(), "attribute"])
        assert repaired == ({"ZipCode"} if spark_ndv else {"Score"}), spark_ndv


def test_band_fallback_through_the_api():
    rng = np.random.default_rng(0)
    n = 5000
    df = pd.DataFrame({"tid": np.arange(n), "wide": ["w%d" % v for v in rng.integers(0, 1000, size=n)],
                       "a": ["a%d" % v for v in rng.integers(0, 5, size=n)],
                       "b": [None if v == 0 else "b%d" % v for v in rng.integers(0, 7, size=n)]})
    rm = _model(df, True, thres=2000)
    rm.run(detect_errors_only=True)
    prov = rm.last_run["distinct_count_provenance"]["columns"]
    assert prov == {"wide": "exact", "a": "estimate", "b": "estimate"}
    assert rm.last_run["detect"].domain_stats["wide"] == df["wide"].nunique()


def test_describe_reports_the_estimates():
    from repair import catalog
    from repair.misc import RepairMisc
    catalog.register("hospital_hll", _hospital())
    try:
        plain = RepairMisc().option("table_name", "hospital_hll").describe()
        est = RepairMisc().option("table_name", "hospital_hll").option("spark_compatible_distinct_counts",
                                                                         "true").describe()
    finally:
        catalog.unregister("hospital_hll")
    got = dict(zip(est["attrName"], est["distinctCnt"]))
    assert {c: got[c] for c in HOSPITAL_DOMAIN_STATS} == HOSPITAL_DOMAIN_STATS
    assert dict(zip(plain["attrName"], plain["distinctCnt"]))["Sample"] == 333
    with pytest.raises(ValueError, match="spark_compatible_distinct_counts"):
        RepairMisc().option("table_name", "x").option("spark_compatible_distinct_counts", "yes").describe()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _summary(rm, out):
    res = rm.last_run["detect"]
    cells = sorted((int(r), a, None if c != c else c, None if v != v else v)
                   for r, a, c, v in zip(out["tid"], out["attribute"], out["current_value"], out["repaired"]))
    return (res.domain_stats, rm.last_run["distinct_count_provenance"], {k: v for k, v in res.pairwise_stats.items()},
            sorted(res.disc_attrs), cells)


def _worker(rank, world, port, backend, out_dir):
    import pickle
    import torch.distributed as td
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    td.init_process_group(backend, rank=rank, world_size=world)
    df = _hospital()
    lo, hi = (len(df) * rank) // world, (len(df) * (rank + 1)) // world
    rm = _model(df.iloc[lo:hi].reset_index(drop=True), True, thres=70).setErrorCells(_given(df))
    rm.setDistributed(True, dev)
    rm.option("model.lgb.n_estimators", "8")
    out = rm.run()
    mine = _summary(rm, out)
    gathered = [None] * world
    td.all_gather_object(gathered, mine)
    if rank == 0:
        with open(os.path.join(out_dir, "sharded.pkl"), "wb") as f:
            pickle.dump(gathered, f)
    td.barrier()
    td.destroy_process_group()


def test_two_ranks_give_the_one_gpu_estimates_and_outputs(tmp_path):
    import pickle
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    mp.spawn(_worker, args=(2, _free_port(), backend, str(tmp_path)), nprocs=2, join=True)
    with open(os.path.join(tmp_path, "sharded.pkl"), "rb") as f:
        parts = pickle.load(f)
    rm = _model(_hospital(), True, thres=70).setErrorCells(_given(_hospital()))
    rm.option("model.lgb.n_estimators", "8")
    want = _summary(rm, rm.run())
    assert want[4] and {a for _, a, _, _ in want[4]} == {"ZipCode"}
    for part in parts:
        assert part[:4] == want[:4]
    assert sorted(c for part in parts for c in part[4]) == want[4]
