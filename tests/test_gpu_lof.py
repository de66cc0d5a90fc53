"""LOFOutlierErrorDetector on the device: dr_lof_score bit for bit against the oracle's weighted
formulation, the reference's known answers through the standalone and pipeline APIs, Arrow input, and a
two-rank sharded run equal to the one-GPU run.  ScikitLearnBackedErrorDetector is checked alongside."""
import os
import socket
import warnings

import numpy as np
import pandas as pd
import pytest

import parity_utils as PU
from oracle import lof as OL

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def _ctx():
    from repair._native import Context
    return Context.acquire(0)


def _score(u, cnt, k):
    ctx = _ctx()
    try:
        d_u = torch.from_numpy(np.asarray(u, dtype=np.float64)).to(DEV)
        d_c = torch.from_numpy(np.asarray(cnt, dtype=np.int64)).to(DEV)
        n = len(u)
        out = [torch.empty(n, dtype=torch.float64, device=DEV) for _ in range(3)]
        verdict = torch.empty(n, dtype=torch.uint8, device=DEV)
        ctx.lof_score(d_u, d_c, k, verdict, out[0], out[1], out[2])
        return [t.cpu().numpy() for t in out] + [verdict.cpu().numpy().astype(bool)]
    finally:
        from repair._native import Context
        Context.release(ctx)


def _entries(case):
    rng = np.random.default_rng(sum(ord(ch) for ch in case))
    if case == "distinct":
        u = np.unique(rng.normal(size=5000))
        return u, np.ones(len(u), dtype=np.int64)
    if case == "heavy_duplicates":       # c_i - 1 >= k for most entries
        u = np.unique(rng.normal(size=300))
        return u, rng.integers(20, 200, size=len(u))
    if case == "partial_runs":
        u = np.unique(rng.normal(size=4000) * 10)
        return u, rng.integers(1, 9, size=len(u))
    if case == "equal_distance_ties":    # evenly spaced: every boundary is a tie
        u = np.arange(-1500, 1500, dtype=np.float64) * 0.25
        return u, rng.integers(1, 4, size=len(u))
    if case == "huge_counts":            # multiplicities of 10^9 rows
        u = np.unique(rng.normal(size=2000))
        c = rng.integers(1, 3, size=len(u))
        c[::7] = 1_000_000_000
        return u, c
    if case == "d_below_k":
        return np.array([-3.0, 0.5, 1.0, 2.0, 40.0]), np.array([3, 1, 10, 2, 5])
    if case == "d_one":
        return np.array([7.25]), np.array([30])
    if case == "many_tiles":             # >= 10^6 entries: halos across CTA tile edges
        u = np.unique(np.round(rng.normal(size=1_300_000) * 1e4, 1))
        return u, rng.integers(1, 4, size=len(u))
    raise KeyError(case)


@pytest.mark.parametrize("case", ["distinct", "heavy_duplicates", "partial_runs", "equal_distance_ties",
                                  "huge_counts", "d_below_k", "d_one", "many_tiles"])
def test_lof_score_bit_identical_to_oracle(case):
    u, cnt = _entries(case)
    k = OL.effective_k(int(np.sum(cnt)))
    want = OL.lof_entries(u, cnt, k)
    got = _score(u, cnt, k)
    for name, g, w in zip(("kdist", "lrd", "lof", "verdict"), got, want):
        assert np.array_equal(g, w), "{}: {} of {} entries differ".format(name, int((g != w).sum()), len(u))
    if case in ("distinct", "partial_runs", "many_tiles"):
        assert got[3].any()


@pytest.mark.parametrize("median_in_dictionary", [True, False])
def test_engine_entries_and_flags_match_oracle(median_in_dictionary):
    from repair.engine import Engine
    from repair.table import EncodedTable
    rng = np.random.default_rng(11)
    # 3701 non-NULL values rounded to 0.1: the median is a cell value; 3700 distinct values: the median
    # is the mean of two cells and no cell holds it
    n = 4001 if median_in_dictionary else 4000
    x = rng.normal(size=n) * 5
    if median_in_dictionary:
        x = np.round(x, 1)
    x[:3] = [80.0, -75.5, 120.0]
    x[rng.choice(np.arange(3, n), 300, replace=False)] = np.nan
    df = pd.DataFrame({"tid": np.arange(len(x)), "v": x, "s": ["a"] * len(x)})
    u, cnt, k, inv = OL.weighted_column(x)
    med = np.median(x[~np.isnan(x)])
    assert (med in set(x[~np.isnan(x)].tolist())) == median_in_dictionary
    enc = EncodedTable.from_pandas(df, "tid")
    engine = Engine(enc, 0)
    try:
        hist = engine.raw_value_counts_dev("v")
        d_u, d_c, k_got, _, inserted = engine.lof_entries(np.asarray(enc.by_name["v"].dictionary), hist)
        assert inserted == (not median_in_dictionary)
        assert k_got == k
        assert np.array_equal(d_u.cpu().numpy(), u) and np.array_equal(d_c.cpu().numpy(), cnt)
        bitmaps = {}
        engine.detect_lof(["v"], bitmaps)
        rows = engine.bitmap_rows(bitmaps["v"]).cpu().numpy()
    finally:
        engine.close()
    verdict = OL.lof_entries(u, cnt, k)[3]
    assert rows.tolist() == np.nonzero(verdict[inv])[0].tolist()
    assert len(rows) >= 3


def _kat_frame(n):
    """The reference's test_errors.py:236-270 table (integer columns with a NULL row, as toPandas gives them)."""
    ids = np.r_[np.arange(n), 1000000, 1000001, 1000002]
    v1 = np.r_[np.arange(n) % 2, 1, 1000, np.nan].astype(np.float64)
    v2 = np.r_[np.arange(n) % 3, 1000, 1, np.nan].astype(np.float64)
    return pd.DataFrame({"id": ids, "v1": v1, "v2": v2})


@pytest.mark.parametrize("n", [3000, 10000])
def test_reference_kat_standalone(n):
    from sklearn.neighbors import LocalOutlierFactor
    from repair.errors import LOFOutlierErrorDetector, ScikitLearnBackedErrorDetector
    df = _kat_frame(n)
    cases = [(["v1", "v2"], [(1000000, "v2"), (1000001, "v1")]), (["v1"], [(1000001, "v1")]),
             (["Unknown", "v1"], [(1000001, "v1")]), (["Non-existent"], [])]
    makers = [lambda: LOFOutlierErrorDetector(5000, num_parallelism=1),
              lambda: ScikitLearnBackedErrorDetector(lambda: LocalOutlierFactor(novelty=False), 5000, 1)]
    for make in makers:
        for targets, want in cases:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                out = make().setUp("id", df, ["v1", "v2"], targets).detect()
            got = sorted((int(i), a) for i, a in zip(out["id"], out["attribute"]))
            assert got == want, (str(make()), targets)


def _boston():
    df = pd.read_csv(os.path.join(GOLDEN, "boston.csv"))
    df["CHAS"] = df["CHAS"].map(lambda v: None if v != v else str(v))
    df["RAD"] = df["RAD"].map(lambda v: None if v != v else str(int(v)) if float(v).is_integer() else str(v))
    return df


def _boston_expected(df):
    """NULL cells of every attribute + the oracle's LOF cells of every numeric attribute, as (tid, attr)."""
    want = set()
    for c in df.columns:
        if c == "tid":
            continue
        for r in np.nonzero(df[c].isna().to_numpy())[0]:
            want.add((str(df["tid"].iloc[r]), c))
        if df[c].dtype.kind in "if":
            got = OL.weighted_column(df[c].to_numpy(dtype=np.float64))
            if got is not None:
                u, cnt, k, inv = got
                for r in np.nonzero(OL.lof_entries(u, cnt, k)[3][inv])[0]:
                    want.add((str(df["tid"].iloc[r]), c))
    return sorted(want)


def _detect(inp, detectors):
    from repair import RepairModel
    rm = RepairModel().setRowId("tid").setErrorDetectors(detectors)
    rm = rm.setArrowInput(inp) if not isinstance(inp, pd.DataFrame) else rm.setInput(inp)
    return rm.run(detect_errors_only=True)


def test_boston_pipeline_cells_equal_oracle():
    from repair.errors import LOFOutlierErrorDetector, NullErrorDetector
    df = _boston()
    out = _detect(df, [NullErrorDetector(), LOFOutlierErrorDetector()])
    got = sorted({(t[0], t[1]) for t in PU.frame_tuples(out, "tid")})
    assert got == _boston_expected(df)
    assert any(a == "CRIM" for _, a in got) and any(a == "LSTAT" for _, a in got)


def test_boston_arrow_input_gives_the_same_cells():
    import pyarrow as pa
    from repair.errors import LOFOutlierErrorDetector, NullErrorDetector
    df = _boston()
    out = _detect(pa.Table.from_pandas(df, preserve_index=False), [NullErrorDetector(), LOFOutlierErrorDetector()])
    out = out.to_pandas() if isinstance(out, pa.Table) else out
    assert sorted({(t[0], t[1]) for t in PU.frame_tuples(out, "tid")}) == _boston_expected(df)


def test_boston_repair_run_repairs_lof_cells():
    from repair import RepairModel
    from repair.errors import LOFOutlierErrorDetector, NullErrorDetector
    df = _boston()
    rm = RepairModel().setInput(df).setRowId("tid").setErrorDetectors([NullErrorDetector(), LOFOutlierErrorDetector()])
    rm.option("model.hp.max_evals", "1")
    rm.option("model.lgb.n_estimators", "8")
    rep = rm.run()
    cont = {c for c in df.columns if c != "tid" and df[c].dtype.kind in "if"}
    fixed = [t for t in PU.frame_tuples(rep, "tid") if t[1] in cont]
    assert len(fixed) > 0 and all(t[-1] is not None for t in fixed)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dist_frame():
    df = _boston()
    rng = np.random.default_rng(5)
    crim = df["CRIM"].to_numpy(dtype=np.float64).copy()
    crim[rng.choice(len(crim), 40, replace=False)] = np.nan   # NULL cells take the median's verdict
    df["CRIM"] = crim
    return df


def _dist_worker(rank, world, port, out_dir):
    import torch.distributed as td
    from sklearn.neighbors import LocalOutlierFactor
    from repair import RepairModel
    from repair.errors import LOFOutlierErrorDetector, NullErrorDetector, ScikitLearnBackedErrorDetector
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    td.init_process_group(backend, rank=rank, world_size=world)
    df = _dist_frame()
    lo, hi = (len(df) * rank) // world, (len(df) * (rank + 1)) // world
    mine = df.iloc[lo:hi].reset_index(drop=True)
    dets = [NullErrorDetector(), LOFOutlierErrorDetector()]
    out = RepairModel().setInput(mine).setRowId("tid").setErrorDetectors(dets).setDistributed(True, dev) \
        .run(detect_errors_only=True)
    got = sorted({(t[0], t[1]) for t in PU.frame_tuples(out, "tid")})
    gathered = [None] * world
    td.all_gather_object(gathered, got)
    mine_ids = {str(t) for t in mine["tid"].tolist()}
    assert all(t in mine_ids for t, _ in got)
    with pytest.raises(NotImplementedError, match="setDistributed"):
        RepairModel().setInput(mine).setRowId("tid").setDistributed(True, dev).setErrorDetectors(
            [ScikitLearnBackedErrorDetector(lambda: LocalOutlierFactor(novelty=False))]).run(detect_errors_only=True)
    if rank == 0:
        union = sorted(t for part in gathered for t in part)
        one = sorted({(t[0], t[1]) for t in PU.frame_tuples(_detect(df, dets), "tid")})
        assert union == one
        assert any(a == "CRIM" for _, a in one)
        assert union == _boston_expected(df)
    td.barrier()
    open(os.path.join(out_dir, "ok%d" % rank), "w").write("ok")
    td.destroy_process_group()


def test_two_rank_lof_equals_one_gpu(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_dist_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert sorted(os.listdir(tmp_path)) == ["ok0", "ok1"]
