"""delphi.misc utilities without a device: the oracle against the reference's known answers
(python/repair/tests/test_misc.py:49-174), the public API's argument checks (raised before any device
work), and the dictionary-code restatement of the k-means assignment against explicit row vectors."""
import os

import numpy as np
import pandas as pd
import pytest

from oracle import misc as OM
from repair import catalog, cluster
from repair.misc import RepairMisc, percentile_hist, target_strings
from repair.table import encode_columns
from repair.utils import AnalysisException

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _adult():
    return pd.read_csv(os.path.join(GOLDEN, "adult.csv"))


def _host_feats(df, targets, q=2):
    cols = {c.name: c for c in encode_columns(df[list(dict.fromkeys(targets))])}
    order = [cols[t] for t in targets]
    hist = [np.bincount(c.codes + 1, minlength=c.dict_size + 1).astype(np.int64) for c in order]
    return cluster.QgramFeatures(target_strings(order), hist, q), order


# ---- known answers ---------------------------------------------------------------------------------------
def test_flatten_known_answer():
    df = pd.DataFrame({"tid": [1, 2, 3], "v": ["a", "b", "c"]})
    got = OM.flatten(df, "tid")
    assert list(got.itertuples(index=False, name=None)) == [(1, "v", "a"), (2, "v", "b"), (3, "v", "c")]


def test_inject_null_ratio_one_known_answer():
    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a", "b", "c", "d"], "v2": [1, 1, 1, 2]})
    got = OM.inject_null(df, {"v1"}, 1.0, seed=123)
    assert got["v1"].tolist() == [None] * 4
    assert got["v2"].tolist() == [1, 1, 1, 2] and got["tid"].tolist() == [1, 2, 3, 4]


def test_to_histogram_known_answer():
    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a"] * 4, "v2": [1, 1, 1, 2]})
    got = OM.to_histogram(df, "v1,v2")
    assert list(got.itertuples(index=False, name=None)) == [("v1", [{"value": "a", "cnt": 4}])]


def test_to_error_map_known_answer():
    df = pd.DataFrame({"tid": [1, 2, 3, 4], "v1": ["a", "b", "c", "d"], "v2": [1, 1, 1, 2]})
    cells = pd.DataFrame({"tid": [1, 2, 4, 4], "attribute": ["v1", "v2", "v1", "v2"]})
    got = OM.to_error_map(df, "tid", cells)
    assert got["error_map"].tolist() == ["*-", "-*", "--", "**"]


ADULT_DESCRIBE = [("Age", 4, None, None, 2, 5, 5, None), ("Country", 3, None, None, 0, 13, 13, None),
                  ("Education", 7, None, None, 0, 9, 12, None), ("Income", 2, None, None, 2, 11, 11, None),
                  ("Occupation", 7, None, None, 0, 13, 17, None), ("Relationship", 4, None, None, 0, 9, 13, None),
                  ("Sex", 2, None, None, 3, 5, 6, None)]
RANGE_DESCRIBE = [("id", 100, None, None, 0, 2, 2, None), ("v1", 9, "0", "8", 0, 8, 8, [0.125] * 8),
                  ("v2", 17, "0.0", "16.0", 0, 8, 8, [0.125] * 8)]


def range_table():
    ids = np.arange(100)
    return pd.DataFrame({"id": [str(i) for i in ids], "v1": ids % 9, "v2": (ids % 17).astype(np.float64)})


def _rows(frame, drop=None):
    out = [tuple(r) for r in frame.itertuples(index=False, name=None) if r[0] != drop]
    return sorted(out, key=lambda r: r[0])


def test_describe_known_answers():
    assert _rows(OM.describe(_adult()), drop="tid") == ADULT_DESCRIBE
    assert _rows(OM.describe(range_table())) == RANGE_DESCRIBE


def test_percentile_hist_rule():
    vals = np.arange(9, dtype=np.float64)
    cnt = np.bincount(np.arange(100) % 9)
    assert percentile_hist(vals, cnt, 8) == [0.125] * 8


def test_split_known_answer_k3_both_algorithms():
    df = _adult()
    targets = [c for c in df.columns if c != "tid"]
    feats, _ = _host_feats(df, targets)
    x, terms = OM.bags(df, targets, 2)
    assert terms == feats.terms
    init = cluster.kmeanspp(x, 3, np.random.default_rng(cluster.SEED))
    labels, _, _ = OM.kmeans(x, init)
    assert sorted(set(labels.tolist())) == [0, 1, 2]
    assert sorted(set(OM.bisecting_kmeans(x, 3).tolist())) == [0, 1, 2]


# ---- argument checks (no device) ---------------------------------------------------------------------------
@pytest.fixture
def registered():
    catalog.register("misc_adult", _adult())
    catalog.register("misc_cells", pd.DataFrame({"tid": [1], "attribute": ["Age"]}))
    catalog.register("misc_bad_cells", pd.DataFrame({"id": [1], "attribute": ["Age"]}))
    yield
    for t in ("misc_adult", "misc_cells", "misc_bad_cells"):
        catalog.unregister(t)


def test_argtype_checks():
    with pytest.raises(TypeError, match="`key` should be provided as str, got int"):
        RepairMisc().option(1, "value")
    with pytest.raises(TypeError, match="`value` should be provided as str, got int"):
        RepairMisc().option("key", 1)
    with pytest.raises(TypeError, match=r"`options` should be provided as dict\[str,str\], got int"):
        RepairMisc().options(1)
    with pytest.raises(TypeError, match=r"got int in keys"):
        RepairMisc().options({"1": "v1", 2: "v2"})
    with pytest.raises(TypeError, match=r"got float in values"):
        RepairMisc().options({"1": "v1", "2": 1.1})


@pytest.mark.parametrize("method,required", [
    ("describe", "table_name"), ("flatten", "table_name, row_id"), ("splitInputTable", "table_name, row_id, k"),
    ("injectNull", "table_name, target_attr_list"), ("toHistogram", "table_name, targets"),
    ("toErrorMap", "table_name, row_id, error_cells")])
def test_required_options(method, required):
    with pytest.raises(ValueError, match="Required options not found: {}$".format(required)):
        getattr(RepairMisc(), method)()


def test_split_option_errors(registered):
    base = {"table_name": "misc_adult", "row_id": "tid"}
    with pytest.raises(ValueError, match="Option 'k' must be an integer, but 'x' found"):
        RepairMisc().options(dict(base, k="x")).splitInputTable()
    with pytest.raises(ValueError, match="Unknown clustering algorithm found: kmeans"):
        RepairMisc().options(dict(base, k="2", clustering_alg="kmeans")).splitInputTable()
    with pytest.raises(ValueError, match="k must be greater than 1"):
        RepairMisc().options(dict(base, k="1")).splitInputTable()
    with pytest.raises(ValueError, match="`q` must be positive, but 0 got"):
        RepairMisc().options(dict(base, k="2", q="0")).splitInputTable()
    with pytest.raises(AnalysisException, match="Columns 'Nope, Nah' do not exist in 'misc_adult'"):
        RepairMisc().options(dict(base, k="2", target_attr_list="Age,Nope,Nah")).splitInputTable()


@pytest.mark.parametrize("ratio", ["0", "0.0", "1.5", "-0.1", "x", "nan"])
def test_null_ratio_out_of_range(registered, ratio):
    misc = RepairMisc().options({"table_name": "misc_adult", "target_attr_list": "Age", "null_ratio": ratio})
    with pytest.raises(ValueError, match=r"Option 'null_ratio' must be a float in \(0.0, 1.0\], but '{}' found"
                       .format(ratio)):
        misc.injectNull()


def test_unknown_columns_and_missing_row_id(registered):
    with pytest.raises(AnalysisException, match="Columns 'Nope' do not exist in 'misc_adult'"):
        RepairMisc().options({"table_name": "misc_adult", "target_attr_list": "Nope"}).injectNull()
    for method, extra in (("flatten", {}), ("splitInputTable", {"k": "2"}),
                          ("toErrorMap", {"error_cells": "misc_cells"})):
        opts = dict({"table_name": "misc_adult", "row_id": "rid"}, **extra)
        if method == "toErrorMap":
            opts["error_cells"] = "misc_cells"
            with pytest.raises(AnalysisException, match="Table 'misc_cells' must have 'rid' and 'attribute' columns"):
                getattr(RepairMisc().options(opts), method)()
            continue
        with pytest.raises(AnalysisException, match=r"Column 'rid' does not exist in 'misc_adult'\.$"):
            getattr(RepairMisc().options(opts), method)()
    with pytest.raises(AnalysisException, match="Table 'misc_bad_cells' must have 'tid' and 'attribute' columns"):
        RepairMisc().options({"table_name": "misc_adult", "row_id": "tid",
                              "error_cells": "misc_bad_cells"}).toErrorMap()


# ---- the assignment restated over dictionary codes -------------------------------------------------------
def _fixtures():
    adult = _adult()
    hosp = pd.read_csv(os.path.join(GOLDEN, "hospital.csv"))
    boston = pd.read_csv(os.path.join(GOLDEN, "boston.csv"))
    return [("adult", adult, [c for c in adult.columns if c != "tid"], 3),
            ("hospital", hosp, [c for c in hosp.columns if c != "tid"], 5),
            ("boston", boston, ["ZN", "CHAS", "RAD", "TAX"], 4),
            ("boston_mixed", boston, ["ZN", "RAD", "TAX", "PTRATIO"], 4)]


@pytest.mark.parametrize("case", ["adult", "hospital", "boston", "boston_mixed"])
def test_code_assignment_equals_row_vectors(case):
    name, df, targets, k = [f for f in _fixtures() if f[0] == case][0]
    feats, cols = _host_feats(df, targets)
    x, terms = OM.bags(df, targets, 2)
    assert terms == feats.terms
    rng = np.random.default_rng(5)
    for centres in (cluster.kmeanspp(x, k, np.random.default_rng(0)), rng.random((k, len(terms)))):
        P, mu_sq = feats.p_table(centres)
        got = OM.assign_from_p([c.codes for c in cols], feats.dom, feats.p_off, P, mu_sq)
        d = OM.sq_dist(x, centres)
        want = np.argmin(d, axis=1)
        for r in np.nonzero(got != want)[0]:
            best = d[r, want[r]]
            assert abs(d[r, got[r]] - best) <= 1e-9 * max(abs(best), 1.0), (case, r)


def test_mixed_numeric_targets_print_as_doubles():
    """array(int, double) has DOUBLE elements in Spark: the int cell 1 gives the q-grams of "1.0"."""
    df = pd.DataFrame({"tid": [0, 1], "i": [1, 20], "d": [0.5, np.nan], "s": ["x", "y"]})
    feats, _ = _host_feats(df, ["i", "d"])
    x, terms = OM.bags(df, ["i", "d"], 2)
    assert terms == feats.terms and {"1.", ".0", "20", "0."} <= set(terms)
    feats, _ = _host_feats(df, ["i", "s"])      # with a string target every column keeps its own text
    assert "1" in feats.terms and ".0" not in feats.terms
    assert OM.bags(df, ["i", "s"], 2)[1] == feats.terms


@pytest.mark.parametrize("bins,msg", [("0", "The number of bins must be greater than 1, but 0 found"),
                                      ("1", "The number of bins must be greater than 1, but 1 found"),
                                      ("x", "Option 'num_bins' must be an integer, but 'x' found")])
def test_num_bins_checked_before_device_work(registered, bins, msg):
    with pytest.raises(ValueError, match=msg):
        RepairMisc().options({"table_name": "misc_adult", "num_bins": bins}).describe()


def test_too_many_split_targets(registered):
    wide = pd.DataFrame({"tid": np.arange(3)})
    for i in range(65):
        wide["c%02d" % i] = ["a", "b", "c"]
    catalog.register("misc_wide", wide)
    try:
        with pytest.raises(ValueError, match="splitInputTable takes at most 64 target columns, but 65 found"):
            RepairMisc().options({"table_name": "misc_wide", "row_id": "tid", "k": "2"}).splitInputTable()
    finally:
        catalog.unregister("misc_wide")
