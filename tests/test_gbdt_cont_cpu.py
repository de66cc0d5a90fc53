"""Continuous targets and features in the GPU trainer's host code: quantile binning (gbdt.bin_sample),
the routing between the GPU trainer and scikit-learn (model.gpu_trainer_bins) and the host-side guards
in front of the device (gbdt.train_gpu, forest.DeviceModel.predict).  No GPU needed."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")


def _cont_sample(n=3000, seed=5):
    """Seeded float64 columns: NULLs, a duplicate-heavy column, a > 254-value column, +-inf, all-NULL and
    single-valued columns."""
    rng = np.random.default_rng(seed)
    cols = {
        "dup": rng.choice([0.5, 1.25, 7.0, -3.0], size=n),
        "wide": rng.normal(size=n) * 100.0,
        "nulls": np.where(rng.random(n) < 0.3, np.nan, rng.integers(0, 40, size=n).astype(np.float64)),
        "inf": np.where(rng.random(n) < 0.1, np.inf, np.where(rng.random(n) < 0.1, -np.inf, rng.normal(size=n))),
        "inf_few": rng.choice([-np.inf, 2.0, 3.5, np.inf, np.nan], size=n),
        "all_null": np.full(n, np.nan),
        "single": np.where(rng.random(n) < 0.2, np.nan, 4.25),
        "huge": rng.choice([1.5e308, 1.7e308, -1.7e308, 0.0], size=n),
    }
    cols["wide"][rng.random(n) < 0.05] = np.nan
    return cols


def _bin(cols, max_bin=255):
    from repair import gbdt as G
    enc = [{"attr": a, "type": "cont"} for a in cols]
    return G.bin_sample(enc, {}, {}, max_bin=max_bin, sample_values=cols)


@pytest.mark.parametrize("max_bin", [255, 16, 2])
def test_continuous_bins_hold_every_sample_value(max_bin):
    from repair import gbdt as G
    cols = _cont_sample()
    bins, n_bins, values = _bin(cols, max_bin)
    max_real = min(255, max(2, max_bin)) - 1
    for f, (a, x) in enumerate(cols.items()):
        b = bins[:, f].astype(np.int64)
        nb = int(n_bins[f])
        assert b.max() < nb
        assert np.all(b[np.isnan(x)] == nb - 1) and np.all(b[~np.isnan(x)] < nb - 1)   # NaN: the missing bin
        assert nb - 1 <= max_real
        distinct = np.unique(x[~np.isnan(x)])
        if len(distinct) <= max_real:                                      # one bin per distinct value
            assert np.array_equal(values[f], distinct) and nb == len(distinct) + 1
            hi = lo = values[f]
        else:
            hi, lo = values[f]
            assert np.all(lo <= hi) and np.all(hi[:-1] < lo[1:])             # disjoint, ordered ranges
        ok = ~np.isnan(x)
        assert np.all((x[ok] >= lo[b[ok]]) & (x[ok] <= hi[b[ok]]))
        # every threshold the trainer can pick (after value bin t < n_real - 1) separates the sample
        n_real = nb - 1
        for t in range(n_real - 1):
            thr = _flat_threshold(values, len(cols), f, t)
            assert np.isfinite(thr) or not np.isfinite(hi[t])
            assert np.all(x[ok & (b <= t)] <= thr) and np.all(x[ok & (b > t)] > thr), (a, t)
    if max_bin == 255:
        assert list(n_bins[[5, 6]]) == [1, 2]                              # all-NULL: one bin; single value: two


def _flat_threshold(values, n_features, f, t):
    """Threshold of a one-split tree on feature f after bin t, through gbdt.flatten."""
    from repair import gbdt as G
    nodes = np.zeros((1, 1, G.MAX_NODES), dtype=G.NODE_DTYPE)
    nodes[0, 0, 0] = (f, t, 0, 1, 2, (0, 0), 0.0)
    nodes[0, 0, 1] = (-1, 0, 0, 0, 0, (0, 0), -1.0)
    nodes[0, 0, 2] = (-1, 0, 0, 0, 0, (0, 0), 1.0)
    return G.flatten(nodes, np.array([[3]]), np.zeros(1), values, n_features, 1)["threshold"][0]


def test_continuous_binning_known_answer():
    x = np.array([3.0, np.nan, 1.0, 3.0, -np.inf, 2.0, 1.0, np.inf])
    bins, n_bins, values = _bin({"x": x})
    assert bins[:, 0].tolist() == [3, 5, 1, 3, 0, 2, 1, 4]
    assert n_bins.tolist() == [6]
    assert values[0].tolist() == [-np.inf, 1.0, 2.0, 3.0, np.inf]
    # midpoints between neighbours; the split bin's largest value where a midpoint is not finite
    assert [_flat_threshold(values, 1, 0, t) for t in range(4)] == [-np.inf, 1.5, 2.5, 3.0]
    # above max_bin - 1 values: equal-count groups of adjacent values, thresholds between the groups
    bins, n_bins, values = _bin({"x": np.array([1.0, 2.0, 3.0, 4.0, 5.0, 6.0, np.nan])}, max_bin=4)
    assert bins[:, 0].tolist() == [0, 0, 1, 1, 2, 2, 3] and n_bins.tolist() == [4]
    assert values[0].tolist() == [[2.0, 4.0, 6.0], [1.0, 3.0, 5.0]]
    assert [_flat_threshold(values, 1, 0, t) for t in range(2)] == [2.5, 4.5]


def test_adjacent_doubles_keep_the_split_exact():
    a = 1.0
    b = np.nextafter(a, 2.0)
    bins, _, values = _bin({"x": np.array([a, b, a, b])})
    thr = _flat_threshold(values, 1, 0, 0)
    assert a <= thr < b


def test_discrete_features_bin_as_before_next_to_continuous_ones():
    from repair import gbdt as G
    from repair.forest import first_seen
    rng = np.random.default_rng(0)
    codes = rng.integers(-1, 600, size=4000)
    enc = [{"attr": "a", "type": "ordinal", "categories": first_seen(codes)}]
    alone = G.bin_sample(enc, {"a": codes}, {"a": 600})
    x = rng.normal(size=4000)
    mixed = G.bin_sample(enc + [{"attr": "c", "type": "cont"}], {"a": codes}, {"a": 600},
                         sample_values={"c": x})
    assert np.array_equal(mixed[0][:, 0], alone[0][:, 0]) and mixed[1][0] == alone[1][0]
    assert np.array_equal(mixed[2][0], alone[2][0])
    # without the float64 values a continuous feature cannot be binned
    assert G.bin_sample(enc + [{"attr": "c", "type": "cont"}], {"a": codes}, {"a": 600}) is None


# ---- routing -------------------------------------------------------------------------------------------
def _route(opts, continuous, n_bins, trainer="gpu"):
    from repair.model import gpu_trainer_bins
    calls = []

    def bin_fn():
        calls.append(1)
        return None if n_bins is None else (None, np.asarray(n_bins, dtype=np.int32), None)
    got = gpu_trainer_bins(trainer, opts, continuous, bin_fn)
    return got is not None, bool(calls)


@pytest.mark.parametrize("opts", [{"model.lgb.boosting_type": "dart"}, {"model.lgb.boosting_type": "goss"},
                                  {"model.lgb.boosting_type": "rf"}, {"model.lgb.reg_alpha": "0.1"},
                                  {"model.lgb.min_split_gain": "0.01"}])
def test_boosting_options_send_continuous_models_to_the_gpu_trainer(opts):
    small = [255] * 13
    assert _route(opts, True, small) == (True, True)
    assert _route(opts, False, small) == (True, True)
    assert _route(opts, True, small, trainer="sklearn") == (False, False)
    assert _route(opts, True, [3] * 129) == (False, True)                 # over 128 encoded features
    assert _route(opts, True, [256, 3]) == (False, True)                  # over 255 bins
    assert _route(opts, True, [255] * 68) == (False, True)                # over the 200 KB histogram budget
    assert _route(opts, True, [255] * 66) == (True, True)
    assert _route(opts, True, None) == (False, True)                      # could not be binned


def test_default_options_keep_continuous_models_on_scikit_learn():
    for opts in ({}, {"model.lgb.boosting_type": "gbdt", "model.lgb.reg_alpha": "0.0",
                      "model.lgb.min_split_gain": "0", "model.lgb.max_bin": "64"}):
        assert _route(opts, True, [10, 20]) == (False, False)             # not even binned
        assert _route(opts, False, [10, 20]) == (True, True)              # all-discrete: the GPU trainer


# ---- guards --------------------------------------------------------------------------------------------
def test_train_gpu_refuses_bad_bins_before_any_device_work():
    from repair import gbdt as G
    rng = np.random.default_rng(2)
    n_bins = np.array([5, 3, 9], dtype=np.int32)
    bins = np.stack([rng.integers(0, nb, size=200) for nb in n_bins], axis=1).astype(np.uint8)
    y = rng.normal(size=200)
    cpu = torch.device("cpu")
    vals = [np.arange(8.0)] * 3

    def run(b, nb):
        G.train_gpu(None, cpu, b, nb, vals, y, 1, np.ones(200), 3, 0.1, 3)
    bad = bins.copy()
    bad[17, 1] = 3                                                         # == n_bins[1]
    with pytest.raises(ValueError, match="feature 1: bin byte 3 >= n_bins 3"):
        run(bad, n_bins)
    bad[17, 1] = 255
    with pytest.raises(ValueError, match="bin byte"):
        run(bad, n_bins)
    with pytest.raises(ValueError, match=r"\[1, 255\]"):
        run(bins, np.array([5, 0, 9], dtype=np.int32))
    with pytest.raises(ValueError, match=r"\[1, 255\]"):
        run(np.zeros((200, 3), dtype=np.uint8), np.array([5, 256, 9], dtype=np.int32))
    with pytest.raises(ValueError, match="one column per n_bins entry"):
        run(bins, n_bins[:2])
    with pytest.raises(ValueError, match="uint8"):
        run(bins.astype(np.int32), n_bins)


def test_regression_scale_keeps_the_hessian_quantum_in_range():
    """A regression's hessian quantum 2^bits / spread / 2^goss_shift stays within [1024, 2^bits]: targets
    outside that window are scaled by a power of two to a spread in [1, 2)."""
    from repair import gbdt as G
    assert G.quant_bits(1000) == 20 and G.quant_bits(9000) == 16
    assert G.regression_scale(np.array([0.0, 4.0]), 2.0, 1000) == 0        # spread 2: run as specified
    assert G.regression_scale(np.array([0.4, 0.6]), 0.5, 1000) == -4       # spread 0.1 -> 1.6: sums fit int32
    y = np.array([-1.2e5, 3.2e5])
    assert G.regression_scale(y, 0.0, 9000) == 18                          # 3.2e5 -> 1.22: quantum 2^16 / 1.22
    assert G.regression_scale(np.array([0.0, 40.0]), 0.0, 9000) == 0       # quantum 1638 >= 1024
    assert G.regression_scale(np.array([0.0, 40.0]), 0.0, 9000, goss_shift=3) == 5   # 204 < 1024: 40 -> 1.25
    assert G.regression_scale(np.array([3.0, 3.0]), 3.0, 1000) == 0        # constant target
    for spread in (0.1, 0.75, 1.0, 3.0, 1e3, 2.0 ** 40, 1e-9):
        k = G.regression_scale(np.array([0.0, spread]), 0.0, 20000)
        q = 2.0 ** G.quant_bits(20000) / np.ldexp(spread, -k)
        assert G.MIN_HESS_QUANTUM <= q <= 2.0 ** G.quant_bits(20000), spread


def _cont_model(kind):
    """A one-split model on a continuous feature (float64 tile column 2) -> DeviceModel on the CPU."""
    from repair.forest import DeviceModel
    forest = {"n_features": 1, "n_classes": 1 if kind == "regressor" else 2, "baseline": np.zeros(1),
              "tree_seq": np.zeros(1, dtype=np.int32), "tree_offset": np.array([0, 3]),
              "feature": np.array([0, -1, -1], dtype=np.int32), "threshold": np.array([0.5, 0.0, 0.0]),
              "missing_left": np.zeros(3, dtype=np.uint8), "left": np.array([1, 0, 0], dtype=np.int32),
              "right": np.array([2, 0, 0], dtype=np.int32), "value": np.array([0.0, -1.0, 1.0])}
    spec = {"forest": forest, "encoders": [{"attr": "c", "type": "cont"}],
            "class_codes": None if kind == "regressor" else [3, 7], "integral": False}
    return DeviceModel(spec, {"y": 0}, {}, {"c": 2, "y": 0}, torch.device("cpu"))


@pytest.mark.parametrize("kind", ["classifier", "regressor"])
def test_predict_refuses_a_continuous_model_without_its_float64_tile(kind):
    dm = _cont_model(kind)
    assert dm.max_ccol == 2
    tile = torch.zeros((4, 1), dtype=torch.int32)
    cells = torch.arange(4, dtype=torch.int32)
    with pytest.raises(ValueError, match="no float64 tile"):
        dm.predict(None, tile, 1, None, 0, cells, 4, 0)
    with pytest.raises(ValueError, match="2 columns"):
        dm.predict(None, tile, 1, torch.zeros((4, 2), dtype=torch.float64), 2, cells, 4, 0)


def test_predict_refuses_a_regressor_without_a_float64_tile():
    from repair.forest import DeviceModel
    forest = {"n_features": 1, "n_classes": 1, "baseline": np.zeros(1), "tree_seq": np.zeros(1, dtype=np.int32),
              "tree_offset": np.array([0, 1]), "feature": np.array([-1], dtype=np.int32), "threshold": np.zeros(1),
              "missing_left": np.zeros(1, dtype=np.uint8), "left": np.zeros(1, dtype=np.int32),
              "right": np.zeros(1, dtype=np.int32), "value": np.array([2.0])}
    spec = {"forest": forest, "encoders": [{"attr": "a", "type": "ordinal", "categories": [0, 1]}],
            "class_codes": None, "integral": False}
    dm = DeviceModel(spec, {"a": 0}, {"a": 2}, {}, torch.device("cpu"))
    assert dm.max_ccol == -1
    with pytest.raises(ValueError, match="regressor"):
        dm.predict(None, torch.zeros((2, 1), dtype=torch.int32), 1, None, 0, torch.arange(2, dtype=torch.int32), 2, 0)
