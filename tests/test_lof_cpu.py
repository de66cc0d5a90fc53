"""LOFOutlierErrorDetector / ScikitLearnBackedErrorDetector without a device: the oracle's weighted
formulation of LocalOutlierFactor against scikit-learn itself, the reference's known answers, and the
constructor contract of the new detector classes."""
import os
import warnings

import numpy as np
import pandas as pd
import pytest

from oracle import lof as OL

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sklearn(vals):
    from sklearn.neighbors import LocalOutlierFactor
    x = np.asarray(vals, dtype=np.float64)
    filled = np.where(np.isnan(x), np.median(x[~np.isnan(x)]), x)
    m = LocalOutlierFactor(novelty=False)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        labels = m.fit_predict(pd.DataFrame({"c": filled}))
    return labels < 0, -m.negative_outlier_factor_


def _oracle(vals):
    u, cnt, k, inv = OL.weighted_column(vals)
    _, _, lof, verdict = OL.lof_entries(u, cnt, k)
    return verdict[inv], lof[inv]


def kat_columns(n):
    """The reference's test_errors.py:236-270 table: id % 2, id % 3 plus three dirty rows."""
    v1 = np.r_[np.arange(n) % 2, 1, 1000, np.nan].astype(np.float64)
    v2 = np.r_[np.arange(n) % 3, 1000, 1, np.nan].astype(np.float64)
    ids = np.r_[np.arange(n), 1000000, 1000001, 1000002]
    return ids, v1, v2


@pytest.mark.parametrize("n", [3000, 10000])
def test_reference_kat_against_oracle(n):
    from oracle.table import OTable
    ids, v1, v2 = kat_columns(n)
    tbl = OTable(["id", "v1", "v2"], ["int", "int", "int"], [ids.astype(np.float64), v1, v2])
    for targets, cells in [(["v1", "v2"], [(1000000, "v2"), (1000001, "v1")]), (["v1"], [(1000001, "v1")]),
                           (["Unknown", "v1"], [(1000001, "v1")]), (["Non-existent"], [])]:
        got = sorted((int(ids[r]), a) for r, a in OL.lof_cells(tbl, "id", ["v1", "v2"], targets))
        assert got == cells, targets
    # scikit-learn agrees on these columns
    for col in (v1, v2):
        assert np.array_equal(_sklearn(col)[0], _oracle(col)[0])


def test_num_parallelism_must_be_positive():
    from repair.errors import LOFOutlierErrorDetector
    with pytest.raises(ValueError, match="`num_parallelism` must be positive, got 0"):
        LOFOutlierErrorDetector(5000, num_parallelism=0)
    with pytest.raises(ValueError, match="`num_parallelism` must be positive, got -2"):
        LOFOutlierErrorDetector(num_parallelism=-2)


@pytest.mark.parametrize("case", ["normal", "nan_outliers", "small", "tiny"])
def test_oracle_matches_sklearn_on_tie_free_data(case):
    rng = np.random.default_rng({"normal": 1, "nan_outliers": 2, "small": 3, "tiny": 4}[case])
    if case == "normal":
        x = rng.normal(size=5000)
    elif case == "nan_outliers":
        x = rng.normal(size=5000) * 3.0 + 10.0
        x[rng.choice(5000, 100, replace=False)] = np.nan
        x[:6] = [40.0, -25.0, 31.5, 60.0, -19.0, 45.25]
    elif case == "small":
        x = rng.normal(size=12)   # k = min(20, n - 1) = 11
    else:
        x = rng.normal(size=3)
    want_lab, want_lof = _sklearn(x)
    got_lab, got_lof = _oracle(x)
    assert np.array_equal(got_lab, want_lab)
    assert np.allclose(got_lof, want_lof, rtol=1e-12, atol=0)
    if case == "nan_outliers":
        assert got_lab[:6].all()


def _boston_numeric():
    df = pd.read_csv(os.path.join(GOLDEN, "boston.csv"))
    return {c: df[c].to_numpy(dtype=np.float64) for c in df.columns if c != "tid" and df[c].dtype.kind in "if"}


def _has_boundary_tie(vals):
    """Some entry's k-th neighbour is chosen between two values at the same distance."""
    u, cnt, k, _ = OL.weighted_column(vals)
    D = len(u)
    for i in range(D):
        need, l, r = k - min(cnt[i] - 1, k), i - 1, i + 1
        while need > 0:
            dl = u[i] - u[l] if l >= 0 else np.inf
            dr = u[r] - u[i] if r < D else np.inf
            if dl == dr:
                return True
            if dl < dr:
                need -= min(cnt[l], need)
                l -= 1
            else:
                need -= min(cnt[r], need)
                r += 1
    return False


def test_oracle_matches_sklearn_on_boston_except_boundary_ties():
    differ = []
    for c, vals in _boston_numeric().items():
        if not np.array_equal(_sklearn(vals)[0], _oracle(vals)[0]):
            differ.append(c)
            assert _has_boundary_tie(vals), c
    # scikit-learn breaks equal-distance ties in KD-tree traversal order: the one column where that
    # changes a label (2 of 506)
    assert differ == ["PTRATIO"]
    vals = _boston_numeric()["PTRATIO"]
    assert int((_sklearn(vals)[0] != _oracle(vals)[0]).sum()) == 2


def test_single_entry_helper_matches_whole_column():
    rng = np.random.default_rng(7)
    x = np.round(rng.normal(size=20000), 2)   # heavy duplicates and exact ties
    u, cnt, k, _ = OL.weighted_column(x)
    kd, lrd, lof, v = OL.lof_entries(u, cnt, k)
    for i in list(range(0, 70)) + list(range(len(u) - 70, len(u))) + rng.choice(len(u), 200).tolist():
        got = OL.lof_entry(u, cnt, k, i)
        assert got == (kd[i], lrd[i], lof[i], bool(v[i]))
    # many entries at once from concatenated neighbourhoods
    idx = np.unique(np.r_[rng.choice(len(u), 500), 0, 1, len(u) - 1])
    flat, s_lo, s_hi, centre = OL.neighbourhoods(len(u), k, idx)
    got = OL.lof_at(u[flat], cnt[flat], s_lo, s_hi, k, centre)
    for g, w in zip(got, (kd, lrd, lof, v)):
        assert np.array_equal(g, w[idx])


def test_oracle_edge_columns():
    assert OL.weighted_column(np.array([np.nan, np.nan, np.nan])) is None
    assert OL.weighted_column(np.array([1.0])) is None
    with pytest.raises(ValueError, match="infinity"):
        OL.weighted_column(np.array([1.0, np.inf, 2.0]))
    # one distinct value: never an outlier
    u, cnt, k, inv = OL.weighted_column(np.array([5.0] * 30 + [np.nan]))
    assert len(u) == 1 and cnt[0] == 31 and not OL.lof_entries(u, cnt, k)[3].any()


def test_detector_classes_contract():
    import repair
    from repair import errors
    from repair.errors import (LOFOutlierErrorDetector, ScikitLearnBackedErrorDetector,
                               ScikitLearnBasedErrorDetector)
    assert repair.LOFOutlierErrorDetector is LOFOutlierErrorDetector
    assert repair.ScikitLearnBackedErrorDetector is ScikitLearnBackedErrorDetector
    with pytest.raises(TypeError):
        ScikitLearnBasedErrorDetector()   # abstract
    d = LOFOutlierErrorDetector()
    assert str(d) == "LOFOutlierErrorDetector()"
    assert (d.parallel_mode_threshold, d.num_parallelism) == (10000, None)
    assert d.spec() == {"type": "lof"}
    d = LOFOutlierErrorDetector(5000, num_parallelism=3)
    assert (d.parallel_mode_threshold, d.num_parallelism) == (5000, 3)
    assert isinstance(d, errors.ErrorDetector)
    d.setUp("id", "t", ["v1", "v2"], ["Unknown", "v1"])
    assert d._targets == ["Unknown", "v1"]

    from sklearn.neighbors import LocalOutlierFactor
    factory = lambda: LocalOutlierFactor(novelty=False)  # noqa: E731
    s = ScikitLearnBackedErrorDetector(factory, 5000, 1)
    assert str(s) == "ScikitLearnBackedErrorDetector()"
    assert s.spec() == {"type": "sklearn", "factory": factory}
    assert (s.parallel_mode_threshold, s.num_parallelism) == (5000, 1)


def test_sklearn_backed_validation_messages():
    from sklearn.neighbors import LocalOutlierFactor
    from repair.errors import ScikitLearnBackedErrorDetector
    with pytest.raises(ValueError, match="`error_detector_cls` should be callable"):
        ScikitLearnBackedErrorDetector(error_detector_cls=1, parallel_mode_threshold=5000, num_parallelism=1)
    with pytest.raises(ValueError,
                       match="An instance that `error_detector_cls` returns should have a `fit_predict` method"):
        ScikitLearnBackedErrorDetector(error_detector_cls=lambda: 1, parallel_mode_threshold=5000, num_parallelism=1)
    with pytest.raises(ValueError, match="`num_parallelism` must be positive, got 0"):
        ScikitLearnBackedErrorDetector(error_detector_cls=lambda: LocalOutlierFactor(novelty=False),
                                       parallel_mode_threshold=5000, num_parallelism=0)
