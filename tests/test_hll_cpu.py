"""Spark-compatible HyperLogLog++ distinct counts: the oracle (oracle/hll.py) against the values the reference
pins, XXH64 against its published vectors and its own scalar form, the estimator's band fallback, and the
host side of the opt-in mode (setter, Spark types recorded at ingest).  No GPU needed."""
import os
import struct

import numpy as np
import pandas as pd
import pytest

from conftest import GOLDEN
from oracle import hll as H

# RepairSuite.scala:156-175 (convertToDiscretizedTable over hospital.csv read without inferSchema: all strings)
HOSPITAL_DOMAIN_STATS = {
    "HospitalOwner": 28, "MeasureName": 63, "Address2": 0, "Condition": 28, "Address3": 0, "PhoneNumber": 72,
    "CountyName": 65, "ProviderNumber": 71, "HospitalName": 68, "Sample": 355, "HospitalType": 13,
    "EmergencyService": 6, "City": 72, "Score": 71, "ZipCode": 67, "Address1": 78, "State": 4, "Stateavg": 74,
    "MeasureCode": 56}


def _count(values, stype):
    values = list(values)
    return H.distinct_count(H.column_registers(values, stype), len(set(values)))


def test_hospital_domain_stats_match_the_reference():
    df = pd.read_csv(os.path.join(GOLDEN, "hospital.csv"), dtype=str)
    got = {c: _count(sorted(set(df[c].dropna())), "string") for c in HOSPITAL_DOMAIN_STATS}
    assert {c: v for c, (v, _) in got.items()} == HOSPITAL_DOMAIN_STATS
    assert all(how == "estimate" for _, how in got.values())
    # ten of them differ from the exact counts
    exact = {c: df[c].nunique() for c in HOSPITAL_DOMAIN_STATS}
    assert sum(exact[c] != v for c, v in HOSPITAL_DOMAIN_STATS.items()) == 10
    assert (exact["ZipCode"], exact["Score"], exact["Sample"]) == (71, 68, 333)


def test_small_table_stats_match_the_reference():
    ids = np.arange(30)
    # RepairSuite.scala:115-129 computeAndGetTableStats: boolean, long, double, string
    assert _count((ids % 2).astype(bool), "boolean")[0] == 2
    assert _count(ids % 3, "long")[0] == 3
    assert _count((ids % 8).astype(np.float64), "double")[0] == 8
    assert _count([str(v) for v in ids % 6], "string")[0] == 6
    # RepairSuite.scala:131-142 computeDomainSizes: four long columns
    assert [_count(ids % k, "long")[0] for k in (3, 8, 6, 9)] == [3, 8, 6, 9]


def test_xxh64_published_vectors():
    assert H.xxh64(b"", 0) == 0xEF46DB3751D8E999
    assert H.xxh64(b"a", 0) == 0xD24EC4F1A98C6E5B
    assert H.xxh64(b"abc", 0) == 0x44BC2CF5AD770999


def test_xxh64_vectorised_equals_scalar_on_every_length():
    rng = np.random.default_rng(5)
    blobs = [rng.integers(0, 256, size=n, dtype=np.uint8).tobytes() for n in range(101)]
    seeds = rng.integers(0, 2 ** 63, size=len(blobs), dtype=np.int64).astype(np.uint64)
    got = H.hash_bytes_many(blobs, seeds)
    assert got.tolist() == [H.xxh64(b, int(s)) for b, s in zip(blobs, seeds)]
    assert H.hash_bytes_many(blobs).tolist() == [H.xxh64(b, 42) for b in blobs]


def test_typed_hashes_equal_the_scalar_form():
    ints = np.array([0, 1, -1, 2 ** 31 - 1, -2 ** 31, 12345], dtype=np.int64)
    for stype in ("int", "long"):
        assert H.hash_values(ints, stype).tolist() == [H.spark_hash(int(v), stype) for v in ints]
    floats = np.array([0.0, -0.0, 1.5, -2.25, np.nan, np.inf, 1e-30], dtype=np.float64)
    for stype in ("float", "double"):
        assert H.hash_values(floats, stype).tolist() == [H.spark_hash(float(v), stype) for v in floats]
    # normalisation: -0.0 hashes as 0.0, every NaN as the canonical NaN
    other_nan = struct.unpack("<d", struct.pack("<Q", 0x7FF0000000000123))[0]
    for stype in ("float", "double"):
        h = H.hash_values(np.array([0.0, -0.0, np.nan, other_nan, -np.nan]), stype)
        assert h[0] == h[1] and h[2] == h[3] == h[4]
    assert H.spark_hash(True, "boolean") == H.xxh64(struct.pack("<i", 1), 42)
    assert H.spark_hash(None, "string", 7) == 7


def test_xxh64_against_the_xxhash_package():
    xxhash = pytest.importorskip("xxhash")
    for n in range(101):
        b = bytes(range(n))
        assert H.xxh64(b, 42) == xxhash.xxh64_intdigest(b, seed=42)


def test_pair_registers_fold_the_struct_hash():
    rng = np.random.default_rng(1)
    xs, ys = ["a", "bé", "ccc"], ["x", "", "日本語の値", "zz"]
    present = rng.random((len(xs) + 1, len(ys) + 1)) < 0.5
    present[0, 0] = True     # (NULL, NULL) hashes to 42
    hx = np.r_[np.uint64(42), H.hash_values(xs, "string")]
    want = []
    for i, j in zip(*np.nonzero(present)):
        seed = H.spark_hash(None if i == 0 else xs[i - 1], "string")
        want.append(H.spark_hash(None if j == 0 else ys[j - 1], "string", seed))
    assert np.array_equal(H.pair_registers(hx, ys, "string", present), H.registers(want))


def test_band_fallback_is_reported():
    vals = ["v%d" % i for i in range(1000)]
    regs = H.column_registers(vals, "string")
    assert H.estimate(regs) == (None, True)
    assert H.distinct_count(regs, 1000) == (1000, "exact")
    # both ends of the band are estimates
    assert H.distinct_count(H.column_registers(vals[:300], "string"), 300)[1] == "estimate"
    big = ["w%d" % i for i in range(20000)]
    assert H.distinct_count(H.column_registers(big, "string"), 20000)[1] == "estimate"


def test_engine_estimator_equals_the_oracle():
    from repair import hll as RH
    rng = np.random.default_rng(3)
    for n in (0, 1, 5, 100, 399, 450, 1000, 2500, 3000, 50000):
        regs = H.registers(rng.integers(0, 2 ** 63, size=n, dtype=np.int64).astype(np.uint64) * np.uint64(2)
                           + rng.integers(0, 2, size=n).astype(np.uint64))
        est, band = H.estimate(regs)
        assert RH.distinct_count(regs, n) == ((n, RH.EXACT) if band else (est, RH.ESTIMATE))


def test_setter_validation_and_default():
    from repair import RepairModel
    rm = RepairModel()
    assert rm.spark_compatible_distinct_counts is False
    assert rm.setSparkCompatibleDistinctCounts(True) is rm and rm.spark_compatible_distinct_counts is True
    with pytest.raises(TypeError, match="`enabled` should be provided as bool, got str"):
        rm.setSparkCompatibleDistinctCounts("true")


def test_ingest_records_the_spark_type():
    from repair import hll as RH
    from repair.table import EncodedTable, encode_columns
    df = pd.DataFrame({"tid": np.arange(4), "i8": np.array([1, 2, 3, 4], dtype=np.int8),
                       "i32": np.array([1, 2, 3, 4], dtype=np.int32), "i64": np.arange(4, dtype=np.int64),
                       "f32": np.ones(4, dtype=np.float32), "f64": np.ones(4), "s": list("abcd")})
    t = EncodedTable.from_pandas(df, "tid")
    assert {c.name: RH.spark_type(c) for c in t.columns} == {"i8": "int", "i32": "int", "i64": "long",
                                                            "f32": "float", "f64": "double", "s": "string"}
    cols = encode_columns(df.assign(b=np.array([True, False, True, True])))
    assert RH.spark_type(cols[-1]) == "boolean"
    # an integer a float64 dictionary cannot hold exactly is refused, naming the column
    with pytest.raises(ValueError, match="column 'big'"):
        RH.value_buffers("big", np.array([2.0 ** 60]), "long", "cpu")
