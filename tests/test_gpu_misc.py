"""delphi.misc on the device: the reference's known answers through the public API (pandas and Arrow
input), dr_kmeans_assign bit for bit against a NumPy sequential sum, splitInputTable against the oracle's
explicit row vectors, and dr_error_map / dr_null_bits / dr_flatten / describe / toHistogram against the
oracle on real and synthetic tables."""
import os

import numpy as np
import pandas as pd
import pytest

from oracle import misc as OM

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
pa = pytest.importorskip("pyarrow")

from repair import catalog  # noqa: E402
from repair.misc import RepairMisc, split_table  # noqa: E402
from repair.synth import SynthSpec, generate_numpy  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def _adult():
    return pd.read_csv(os.path.join(GOLDEN, "adult.csv"))


def _hospital():
    return pd.read_csv(os.path.join(GOLDEN, "hospital.csv"))


def _boston():
    return pd.read_csv(os.path.join(GOLDEN, "boston.csv"))


_SYNTH = {}


def _synth(n=1_000_000, n_cols=4):
    """1M-row synthetic table of repair/synth.py: string columns c00.. plus an int and a float column."""
    if (n, n_cols) not in _SYNTH:
        codes = generate_numpy(SynthSpec(n, n_cols, null_ratio=0.01, seed=3))
        words = np.array(["v%03d" % i for i in range(64)] + [None], dtype=object)
        df = pd.DataFrame({"tid": np.arange(n, dtype=np.int64)})
        for i, c in enumerate(codes):
            df["c%02d" % i] = words[np.where(c < 0, 64, c)]
        df["num"] = (codes[0].astype(np.int64) * 7) % 23
        df["real"] = np.where(codes[1] < 0, np.nan, codes[1] * 0.5)
        _SYNTH[(n, n_cols)] = df
    return _SYNTH[(n, n_cols)]


def _run(method, df, opts, arrow=False, **kw):
    name = "gpu_misc_input"
    catalog.register(name, pa.Table.from_pandas(df, preserve_index=False) if arrow else df)
    try:
        return getattr(RepairMisc().options(dict(opts, table_name=name)), method)(**kw)
    finally:
        catalog.unregister(name)


def _pandas(out):
    return out.to_pandas() if isinstance(out, pa.Table) else out


# ---- known answers (python/repair/tests/test_misc.py:49-174) -----------------------------------------------
@pytest.mark.parametrize("arrow", [False, True])
def test_known_answers(arrow):
    df = pd.DataFrame({"tid": [1, 2, 3], "v": ["a", "b", "c"]})
    out = _run("flatten", df, {"row_id": "tid"}, arrow)
    assert isinstance(out, pa.Table) == arrow
    out = _pandas(out)
    assert [(int(a), b, c) for a, b, c in zip(out["tid"], out["attribute"].astype(str), out["value"].astype(str))] == \
        [(1, "v", "a"), (2, "v", "b"), (3, "v", "c")]

    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a", "b", "c", "d"], "v2": [1, 1, 1, 2]})
    out = _pandas(_run("injectNull", df, {"target_attr_list": "v1", "null_ratio": "1.0"}, arrow))
    assert out["v1"].isna().all() and out["v2"].tolist() == [1, 1, 1, 2] and out["tid"].tolist() == [1, 2, 3, 4]

    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a"] * 4, "v2": [1, 1, 1, 2]})
    out = _run("toHistogram", df, {"targets": "v1,v2"}, arrow)
    assert list(out.itertuples(index=False, name=None)) == [("v1", [{"value": "a", "cnt": 4}])]

    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a", "b", "c", "d"], "v2": [1, 1, 1, 2]})
    catalog.register("gpu_misc_cells", pd.DataFrame({"tid": [1, 2, 4, 4], "attribute": ["v1", "v2", "v1", "v2"]}))
    try:
        out = _pandas(_run("toErrorMap", df, {"row_id": "tid", "error_cells": "gpu_misc_cells"}, arrow))
    finally:
        catalog.unregister("gpu_misc_cells")
    assert out["error_map"].tolist() == ["*-", "-*", "--", "**"]

    from test_misc_cpu import ADULT_DESCRIBE, RANGE_DESCRIBE, _rows, range_table
    assert _rows(_run("describe", _adult(), {}, arrow), drop="tid") == ADULT_DESCRIBE
    assert _rows(_run("describe", range_table(), {}, arrow)) == RANGE_DESCRIBE

    for alg in ("bisect-kmeans", "kmeans++"):
        out = _pandas(_run("splitInputTable", _adult(), {"row_id": "tid", "k": "3", "clustering_alg": alg}, arrow))
        assert sorted(set(out["k"].tolist())) == [0, 1, 2]


# ---- dr_kmeans_assign ----------------------------------------------------------------------------------------
def _assign_case(n, doms, k, seed, split_mode, ties):
    from repair._native import Context
    rng = np.random.default_rng(seed)
    codes = [np.where(rng.random(n) < 0.05, -1, rng.integers(0, d, n)).astype(np.int32) for d in doms]
    p_off = np.concatenate([[0], np.cumsum([d + 1 for d in doms])[:-1]]).astype(np.int64)
    P = rng.normal(size=(int(sum(d + 1 for d in doms)), k))
    mu_sq = rng.random(k) * 4
    if ties:                     # whole-table ties: equal columns, and small integers that tie per row
        P[:, 1] = P[:, 0]
        mu_sq[1] = mu_sq[0]
        P[:, 2:] = rng.integers(-2, 3, size=(P.shape[0], k - 2)).astype(np.float64)
        mu_sq[2:] = rng.integers(0, 3, size=k - 2)
    labels = split = None
    if split_mode:
        n_labels = k
        labels = rng.integers(-1, n_labels + 1, n).astype(np.int32)
        split = np.full(n_labels, -1, dtype=np.int32)
        split[0] = 2
        split[3 % n_labels] = 4 % k
        split[1] = k - 1                       # s + 1 == k: out of range, rows stay
    want = OM.assign_from_p(codes, doms, p_off, P, mu_sq, labels, split)
    ctx = Context.acquire(0)
    try:
        d_cols = [torch.from_numpy(c).to(DEV) for c in codes]
        d_lab = torch.from_numpy(labels if labels is not None else np.zeros(n, dtype=np.int32)).to(DEV)
        d_split = None if split is None else torch.from_numpy(split).to(DEV)
        ctx.kmeans_assign(d_cols, doms, p_off, n, torch.from_numpy(P).to(DEV), torch.from_numpy(mu_sq).to(DEV),
                          d_lab, d_split)
        got = d_lab.cpu().numpy()
    finally:
        Context.release(ctx)
    return got, want


@pytest.mark.parametrize("split_mode", [False, True])
@pytest.mark.parametrize("shape", ["smem", "global", "many_centres", "ties"])
def test_kmeans_assign_bit_identical(shape, split_mode):
    n = 1_000_003
    if shape == "smem":
        got, want = _assign_case(n, [3, 17, 64, 5, 200], 8, 1, split_mode, False)
    elif shape == "global":                  # P of 4 005 x 8 doubles: 250 KB, above the shared-memory budget
        got, want = _assign_case(n, [4000, 2], 8, 2, split_mode, False)
    elif shape == "many_centres":            # 13 centres: two accumulation passes
        got, want = _assign_case(n, [30, 40, 7], 13, 3, split_mode, False)
    else:
        got, want = _assign_case(n, [5, 9, 3], 6, 4, split_mode, True)
    assert np.array_equal(got, want)


def test_kmeans_assign_unaligned_tail():
    from repair._native import Context
    rng = np.random.default_rng(9)
    n, doms, k = 1001, [4, 6], 3
    base = rng.integers(0, 4, n + 1).astype(np.int32)
    col2 = rng.integers(-1, 6, n + 1).astype(np.int32)
    p_off = np.array([0, 5], dtype=np.int64)
    P = rng.normal(size=(12, k))
    mu_sq = rng.random(k)
    want = OM.assign_from_p([base[1:], col2[1:]], doms, p_off, P, mu_sq)
    ctx = Context.acquire(0)
    try:
        a, b = torch.from_numpy(base).to(DEV), torch.from_numpy(col2).to(DEV)
        lab = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
        ctx.kmeans_assign([a[1:], b[1:]], doms, p_off, n, torch.from_numpy(P).to(DEV),
                          torch.from_numpy(mu_sq).to(DEV), lab[1:])
        got = lab[1:].cpu().numpy()
    finally:
        Context.release(ctx)
    assert np.array_equal(got, want)


# ---- splitInputTable against the oracle ---------------------------------------------------------------------
def _split_cases():
    hosp = _hospital()
    syn = _synth()
    return {"adult": (_adult(), [c for c in _adult().columns if c != "tid"], 3),
            "hospital": (hosp, [c for c in hosp.columns if c != "tid"], 4),
            "synthetic_1m": (syn, ["c00", "c01", "c02", "c03"], 5)}


@pytest.mark.parametrize("alg", ["bisect-kmeans", "kmeans++"])
@pytest.mark.parametrize("case", ["adult", "hospital", "synthetic_1m"])
def test_split_equals_oracle(case, alg):
    df, targets, k = _split_cases()[case]
    info = {}
    got = split_table(df, targets, k, 2, alg, info)
    x, terms = OM.bags(df, targets, 2)
    if alg == "bisect-kmeans":               # k-means (the reference's crossed names)
        want, iters, _ = OM.kmeans(x, info["init_centres"])
        assert iters == info["iterations"]
    else:
        want = OM.bisecting_kmeans(x, k)
    assert np.array_equal(got, want), (case, alg, int((got != want).sum()))
    assert len(set(got.tolist())) == k


def _wide_table():
    """60 000 rows whose column `w` has 20 000 distinct values: (k + 1)(values + 1) exceeds dr_cooc's 65 535-entry
    tables for every k >= 3, so its centre counts go through dr_label_counts."""
    rng = np.random.default_rng(11)
    n = 60_000
    ids = rng.permutation(n) % 20_000
    return pd.DataFrame({"tid": np.arange(n), "w": ["w%05d" % (i * 7919 % 100_000) for i in ids],
                         "g": np.array(["alpha", "beta", "gamma", None], dtype=object)[rng.integers(0, 4, n)],
                         "h": rng.integers(0, 9, n)})


@pytest.mark.parametrize("alg", ["bisect-kmeans", "kmeans++"])
@pytest.mark.parametrize("k", [3, 8])
def test_split_high_cardinality_equals_oracle(k, alg):
    df = _wide_table()
    targets = ["w", "g", "h"]
    assert (k + 1) * (df["w"].nunique() + 1) > 65535
    info = {}
    got = split_table(df, targets, k, 2, alg, info)
    x, _ = OM.bags(df, targets, 2)
    if alg == "bisect-kmeans":
        want, iters, _ = OM.kmeans(x, info["init_centres"])
        assert iters == info["iterations"]
    else:
        want = OM.bisecting_kmeans(x, k)
    assert np.array_equal(got, want), (k, alg, int((got != want).sum()))
    assert len(set(got.tolist())) == k


def test_label_counts_equals_bincount():
    from repair._native import Context
    rng = np.random.default_rng(4)
    n, dom = 1_000_003, 70_000
    labels = rng.integers(0, 12, n).astype(np.int32)
    col = np.where(rng.random(n) < 0.03, -1, rng.integers(0, dom, n)).astype(np.int32)
    col[:5] = dom + 3                                    # out-of-range codes clamp to the last slot
    lo, hi = 4, 10
    ctx = Context.acquire(0)
    try:
        out = torch.zeros((hi - lo, dom + 1), dtype=torch.int64, device=DEV)
        ctx.label_counts(torch.from_numpy(labels).to(DEV), torch.from_numpy(col).to(DEV), dom, n, lo, hi, out)
        got = out.cpu().numpy()
    finally:
        Context.release(ctx)
    m = (labels >= lo) & (labels < hi)
    slot = np.minimum(col.astype(np.int64) + 1, dom)
    want = np.bincount((labels[m] - lo).astype(np.int64) * (dom + 1) + slot[m],
                       minlength=(hi - lo) * (dom + 1)).reshape(hi - lo, dom + 1)
    assert np.array_equal(got, want)


def test_split_api_arrow_equals_pandas():
    df = _hospital()
    opts = {"row_id": "tid", "k": "4", "target_attr_list": "City,State,HospitalName"}
    a = _run("splitInputTable", df, opts, False)
    b = _run("splitInputTable", df, opts, True)
    assert isinstance(b, pa.Table) and b.column_names == ["tid", "k"]
    assert a["k"].tolist() == b.column("k").to_pylist()


# ---- error map, NULL injection, flatten ------------------------------------------------------------------
def _error_cells(df, seed):
    rng = np.random.default_rng(seed)
    attrs = [c for c in df.columns if c != "tid"]
    m = min(len(df) * 2, 200_000)
    cells = pd.DataFrame({"tid": rng.integers(-5, len(df) + 5, m), "attribute":
                          np.array(attrs + ["nope"], dtype=object)[rng.integers(0, len(attrs) + 1, m)]})
    return cells


@pytest.mark.parametrize("case", ["hospital", "synthetic_1m"])
@pytest.mark.parametrize("arrow", [False, True])
def test_error_map_equals_oracle(case, arrow):
    df = _hospital() if case == "hospital" else _synth()
    cells = _error_cells(df, 1)
    if case == "hospital":
        cells = pd.concat([cells, pd.read_csv(os.path.join(GOLDEN, "hospital_error_cells.csv"))[["tid", "attribute"]]])
    catalog.register("gpu_misc_cells", cells)
    try:
        out = _pandas(_run("toErrorMap", df, {"row_id": "tid", "error_cells": "gpu_misc_cells"}, arrow))
    finally:
        catalog.unregister("gpu_misc_cells")
    want = OM.to_error_map(df, "tid", cells)
    assert out["tid"].tolist() == want["tid"].tolist()
    assert out["error_map"].tolist() == want["error_map"].tolist()


def _keep_bits(df, col, seed, ratio):
    ci = list(df.columns).index(col)
    return OM.inject_null_keep(seed, ci, len(df), ratio)


@pytest.mark.parametrize("case", ["hospital", "synthetic_1m"])
@pytest.mark.parametrize("ratio", [0.3, 1.0])
def test_inject_null_equals_oracle_pandas(case, ratio):
    df = _hospital() if case == "hospital" else _synth()
    targets = ["City", "Address2", "Sample"] if case == "hospital" else ["c00", "c02", "num", "real"]
    out = _run("injectNull", df, {"target_attr_list": ",".join(targets), "null_ratio": str(ratio)}, _seed=77)
    for c in df.columns:
        if c not in targets:
            pd.testing.assert_series_equal(out[c], df[c])
            continue
        keep = _keep_bits(df, c, 77, ratio) & df[c].notna().to_numpy()
        assert np.array_equal(out[c].notna().to_numpy(), keep), c
        assert out[c][keep].astype(str).tolist() == df[c][keep].astype(str).tolist()
        if ratio < 1 and len(df) >= 10 ** 6:
            n = len(df)
            hit = (~_keep_bits(df, c, 77, ratio)).sum()
            assert abs(hit - ratio * n) <= 5 * np.sqrt(n * ratio * (1 - ratio))


@pytest.mark.parametrize("offset", [0, 13, 77])
def test_inject_null_arrow_bit_offset(offset):
    df = _synth()
    tbl = pa.Table.from_pandas(df, preserve_index=False)
    n = len(df) - 2 * offset
    sliced = tbl.slice(offset, n)
    # several chunks, each with its own offset
    sliced = pa.concat_tables([sliced.slice(0, n // 3), sliced.slice(n // 3)])
    targets = ["c01", "num", "real"]
    catalog.register("gpu_misc_arrow", sliced)
    try:
        out = RepairMisc().options({"table_name": "gpu_misc_arrow", "target_attr_list": ",".join(targets),
                                    "null_ratio": "0.25"}).injectNull(_seed=5)
    finally:
        catalog.unregister("gpu_misc_arrow")
    assert isinstance(out, pa.Table) and out.schema == sliced.schema
    base = df.iloc[offset:offset + n].reset_index(drop=True)
    for c in targets:
        ci = list(df.columns).index(c)
        keep = OM.inject_null_keep(5, ci, n, 0.25) & base[c].notna().to_numpy()
        col = out.column(c)
        assert np.array_equal(np.asarray(col.is_valid()), keep), c
        assert col.filter(pa.array(keep)).to_pylist() == sliced.column(c).filter(pa.array(keep)).to_pylist()
    assert out.column("c00").equals(sliced.column("c00"))


def test_inject_null_dictionary_arrow_ratio_one():
    df = _hospital()
    tbl = pa.Table.from_pandas(df, preserve_index=False)
    tbl = tbl.set_column(tbl.schema.get_field_index("City"), "City", tbl.column("City").dictionary_encode())
    catalog.register("gpu_misc_arrow", tbl.slice(3))
    try:
        out = RepairMisc().options({"table_name": "gpu_misc_arrow", "target_attr_list": "",
                                    "null_ratio": "1.0"}).injectNull(_seed=1)
    finally:
        catalog.unregister("gpu_misc_arrow")
    assert all(out.column(i).null_count == out.num_rows for i in range(out.num_columns))
    assert pa.types.is_dictionary(out.schema.field("City").type)


def _nulls_as_none(vals):
    """pandas may hold a NULL string as NaN."""
    return [None if v is None or (isinstance(v, float) and v != v) else v for v in vals]


@pytest.mark.parametrize("case", ["hospital", "synthetic_1m"])
@pytest.mark.parametrize("arrow", [False, True])
def test_flatten_equals_oracle(case, arrow):
    df = _hospital() if case == "hospital" else _synth()
    out = _run("flatten", df, {"row_id": "tid"}, arrow)
    want = OM.flatten(df, "tid")
    if arrow:
        assert pa.types.is_dictionary(out.schema.field("value").type)
        assert pa.types.is_dictionary(out.schema.field("attribute").type)
        tid = out.column("tid").to_numpy()
        attr = out.column("attribute").to_pylist()
        val = out.column("value").to_pylist()
    else:
        tid, attr, val = out["tid"].to_numpy(), out["attribute"].tolist(), out["value"].tolist()
    assert np.array_equal(tid, want["tid"].to_numpy())
    assert attr == want["attribute"].tolist()
    assert _nulls_as_none(val) == _nulls_as_none(want["value"].tolist())


def test_flatten_string_row_ids_arrow_offset():
    df = _adult()
    df["tid"] = ["r%d" % i for i in df["tid"]]
    tbl = pa.Table.from_pandas(df, preserve_index=False).slice(5)
    catalog.register("gpu_misc_arrow", tbl)
    try:
        out = RepairMisc().options({"table_name": "gpu_misc_arrow", "row_id": "tid"}).flatten()
    finally:
        catalog.unregister("gpu_misc_arrow")
    want = OM.flatten(df.iloc[5:].reset_index(drop=True), "tid")
    assert out.column("tid").to_pylist() == want["tid"].tolist()
    assert out.column("value").to_pylist() == _nulls_as_none(want["value"].tolist())


# ---- describe / toHistogram -------------------------------------------------------------------------------------
def _cmp_frames(got, want):
    assert list(got.columns) == list(want.columns)
    for g, w in zip(got.itertuples(index=False, name=None), want.itertuples(index=False, name=None)):
        assert g == w or (g[:-1] == w[:-1] and np.allclose(g[-1], w[-1], equal_nan=True)), (g, w)


@pytest.mark.parametrize("case", ["hospital", "boston", "synthetic_1m"])
@pytest.mark.parametrize("arrow", [False, True])
def test_describe_and_histogram_equal_oracle(case, arrow):
    df = {"hospital": _hospital, "boston": _boston, "synthetic_1m": _synth}[case]()
    for bins in ("8", "5"):
        _cmp_frames(_run("describe", df, {"num_bins": bins}, arrow), OM.describe(df, int(bins)))
    targets = ",".join(list(df.columns) + ["nope"])
    _cmp_frames(_run("toHistogram", df, {"targets": targets}, arrow), OM.to_histogram(df, targets))
