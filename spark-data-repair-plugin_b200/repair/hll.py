"""Spark-compatible distinct counts (opt-in: ``RepairModel.setSparkCompatibleDistinctCounts``, the
``spark_compatible_distinct_counts`` option of ``delphi.misc``).

The reference takes every distinct count that drives a decision from Spark's HyperLogLog++ with relative
SD 0.05 (p = 9, 512 registers): ``domain_stats`` (computeColumnStats, RepairApi.scala:108-118), the pair
scores ``approx_count_distinct(struct(x, y))`` (:430-437) and describe's ``distinctCnt``.  The registers are
built on the GPU (csrc/hll.cu) from the dictionaries -- registers are idempotent under max, so the set of
distinct values (or, for a pair, its presence bits) is all they need -- and the estimate is taken here from
the 512 registers.

Spark subtracts an empirical bias from the HLL++ paper's tables when the linear-counting estimate is above
400 and the raw estimate below 5 m = 2560 (true cardinalities of roughly 400 - 2600).  Those tables are not
part of this project: in that band the exact count is used, and the caller records it as a fallback.

The hash depends on the Spark type of the column, taken from the input's dtype as Spark would map it
(``Column.spark_type``): int8 / int16 / int32 -> IntegerType, int64 -> LongType, float32 -> FloatType,
float64 -> DoubleType, bool -> BooleanType, strings -> StringType.  A reference run that read a CSV with
``inferSchema`` saw IntegerType for integral columns that fit 32 bits: pass such a column as int32.
"""
import math

import numpy as np

from ._native import DR_HLL_KIND

P = 9
M = 1 << P
LINEAR_COUNTING_THRESHOLD = 400     # HyperLogLogPlusPlusHelper.THRESHOLDS(p - 4) for p = 9
RAW_ESTIMATE_FLOOR = 5 * M
ALPHA_M2 = 0.7213 / (1.0 + 1.079 / M) * M * M
ESTIMATE, EXACT = "estimate", "exact"
_EXACT_INT_LIMIT = 2.0 ** 53


def spark_type(col):
    """The Spark type a column's values are hashed as (recorded at ingest; the kind's widest type otherwise)."""
    t = getattr(col, "spark_type", None)
    if t is not None:
        return t
    return {"str": "string", "int": "long", "float": "double"}[col.kind]


def distinct_count(regs, exact):
    """Spark's rounded HLL++ estimate from uint8 / int registers -> (count, ESTIMATE), or (exact, EXACT) in the
    bias-table band."""
    regs = np.asarray(regs, dtype=np.int64)
    zeros = int(np.count_nonzero(regs == 0))
    if zeros > 0:
        h = M * math.log(M / zeros)
        if h <= LINEAR_COUNTING_THRESHOLD:
            return int(math.floor(h + 0.5)), ESTIMATE
    e = ALPHA_M2 / float(np.sum(np.ldexp(1.0, -regs)))
    if e >= RAW_ESTIMATE_FLOOR:
        return int(math.floor(e + 0.5)), ESTIMATE
    return int(exact), EXACT


def value_buffers(name, values, stype, device):
    """Non-NULL values of one Spark type -> (kind, device data, device int64 offsets or None, n) as
    dr_hll_dict takes them.  Strings travel as UTF-8 bytes in Arrow layout (8-byte aligned, padded)."""
    import torch
    n = len(values)
    if stype == "string":
        blobs = [str(v).encode("utf-8") for v in values]
        off = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([len(b) for b in blobs], out=off[1:])
        raw = np.frombuffer(b"".join(blobs) + bytes(8), dtype=np.uint8)
        return (DR_HLL_KIND[stype], torch.from_numpy(raw.copy()).to(device), torch.from_numpy(off).to(device), n)
    if stype == "boolean":
        host = np.array([1 if (v is True or str(v).lower() == "true" or v == 1) else 0 for v in values], dtype=np.int32)
    else:
        vals = np.asarray(values, dtype=np.float64)
        if stype in ("int", "long"):
            if n and float(np.max(np.abs(vals))) > _EXACT_INT_LIMIT:
                raise ValueError("column '{}' holds an integer beyond +-2^53 that its float64 dictionary cannot hash "
                                 "exactly for Spark-compatible distinct counts".format(name))
            host = vals.astype(np.int32 if stype == "int" else np.int64)
        else:
            host = vals.astype(np.float32 if stype == "float" else np.float64)
    return DR_HLL_KIND[stype], torch.from_numpy(np.ascontiguousarray(host)).to(device), None, n


def column_registers(ctx, device, name, values, stype, hashes=False):
    """-> (host uint8[512] registers, device uint64 hashes of the entries or None)."""
    import torch
    kind, data, off, n = value_buffers(name, values, stype, device)
    regs = torch.zeros(M, dtype=torch.int32, device=device)
    hx = torch.empty(max(n, 1), dtype=torch.uint64, device=device) if hashes else None
    ctx.hll_dict(kind, data, off, n, regs, hx)
    return regs.cpu().numpy().astype(np.uint8), hx


def column_counts(ctx, device, columns):
    """{name: (count, ESTIMATE | EXACT)} of encoded columns (their dictionaries hold the distinct values)."""
    out = {}
    for c in columns:
        regs, _ = column_registers(ctx, device, c.name, c.dictionary, spark_type(c))
        out[c.name] = distinct_count(regs, c.dict_size)
    return out
