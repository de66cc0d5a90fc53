"""Spark's HyperLogLog++ distinct counts (``HyperLogLogPlusPlusHelper``, relative SD 0.05 -> p = 9), the
judge of csrc/hll.cu.

Restated from the public specifications:

* hash: ``XxHash64Function.hash(value, type, seed = 42)``, i.e. standard XXH64 over the UTF-8 bytes of a
  string, over 4 little-endian bytes for byte / short / int / boolean (0 / 1) and float (``floatToIntBits``),
  over 8 bytes for long and double (``doubleToLongBits``).  Floats are normalised first: -0.0 -> 0.0 and
  every NaN -> the canonical NaN (Spark 3.x; not pinned by a reference test).
* struct: ``hash(struct(a, b)) = hash(b, seed = hash(a, seed = 42))``; a NULL field passes its seed through
  (not pinned by a reference test).
* registers: ``idx = x >>> 55``, ``M[idx] = max(M[idx], nlz((x << 9) | (1 << 8)) + 1)``.
* estimate: linear counting ``m ln(m / V)`` while it is <= 400, the raw estimate ``alpha m^2 / sum 2^-M``
  from 5 m = 2560 on.  In between Spark subtracts an empirical bias from the HLL++ paper's tables, which
  this project does not carry: there the exact count is used and reported as a fallback.

Registers are idempotent under max, so a column's registers are a function of its SET of distinct values;
the functions here take dictionaries (distinct values) and presence matrices (distinct pairs).
"""
import math
import struct

import numpy as np

P = 9
M = 1 << P
SEED = 42
LINEAR_COUNTING_THRESHOLD = 400     # HyperLogLogPlusPlusHelper.THRESHOLDS(p - 4) for p = 9
RAW_ESTIMATE_FLOOR = 5 * M          # below it Spark would subtract the bias tables
ALPHA_M2 = 0.7213 / (1.0 + 1.079 / M) * M * M

SPARK_TYPES = ("string", "int", "long", "float", "double", "boolean")

_MASK = (1 << 64) - 1
P1, P2, P3, P4, P5 = (11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579,
                      2870177450012600261)


# ---- scalar XXH64 (the specification, one value at a time) ---------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _MASK


def _round(acc, lane):
    return (_rotl((acc + lane * P2) & _MASK, 31) * P1) & _MASK


def _fmix(h):
    h ^= h >> 33
    h = (h * P2) & _MASK
    h ^= h >> 29
    h = (h * P3) & _MASK
    return h ^ (h >> 32)


def xxh64(data, seed=SEED):
    """Standard XXH64 of `data` (bytes) as an unsigned 64-bit int."""
    seed &= _MASK
    n, p = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & _MASK, (seed + P2) & _MASK, seed, (seed - P1) & _MASK]
        while p + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], int.from_bytes(data[p + 8 * k:p + 8 * k + 8], "little"))
            p += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _MASK
        for k in range(4):
            h = ((h ^ _round(0, v[k])) * P1 + P4) & _MASK
    else:
        h = (seed + P5) & _MASK
    h = (h + n) & _MASK
    while p + 8 <= n:
        h ^= _round(0, int.from_bytes(data[p:p + 8], "little"))
        h = (_rotl(h, 27) * P1 + P4) & _MASK
        p += 8
    if p + 4 <= n:
        h ^= (int.from_bytes(data[p:p + 4], "little") * P1) & _MASK
        h = (_rotl(h, 23) * P2 + P3) & _MASK
        p += 4
    while p < n:
        h ^= (data[p] * P5) & _MASK
        h = (_rotl(h, 11) * P1) & _MASK
        p += 1
    return _fmix(h)


def value_bytes(value, spark_type):
    """The bytes XxHash64Function hashes for a non-NULL value of a Spark type."""
    if spark_type == "string":
        return str(value).encode("utf-8")
    if spark_type in ("int", "boolean"):
        return struct.pack("<i", int(value))
    if spark_type == "long":
        return struct.pack("<q", int(value))
    if spark_type == "float":
        f = float(value)
        f = 0.0 if f == 0.0 else f
        return struct.pack("<I", 0x7FC00000) if f != f else struct.pack("<f", f)
    if spark_type == "double":
        d = float(value)
        d = 0.0 if d == 0.0 else d
        return struct.pack("<Q", 0x7FF8000000000000) if d != d else struct.pack("<d", d)
    raise ValueError("unknown Spark type {!r}".format(spark_type))


def spark_hash(value, spark_type, seed=SEED):
    """XxHash64Function.hash(value, type, seed); a NULL (None) returns the seed."""
    if value is None:
        return seed & _MASK
    return xxh64(value_bytes(value, spark_type), seed)


# ---- vectorised XXH64 (same function over arrays; per-element seeds) -----------------------------------
_U = np.uint64


def _vrotl(x, r):
    return (x << _U(r)) | (x >> _U(64 - r))


def _vround(acc, lane):
    return _vrotl(acc + lane * _U(P2), 31) * _U(P1)


def _vfmix(h):
    h = h ^ (h >> _U(33))
    h = h * _U(P2)
    h = h ^ (h >> _U(29))
    h = h * _U(P3)
    return h ^ (h >> _U(32))


def _xxh64_rows(mat, seeds):
    """XXH64 of every row of a uint8 matrix [n, L] (all rows L bytes) with per-row uint64 seeds."""
    n, L = mat.shape
    with np.errstate(over="ignore"):
        padded = np.zeros((n, (L + 7) // 8 * 8), dtype=np.uint8)
        padded[:, :L] = mat
        words = padded.view("<u8")
        p = 0
        if L >= 32:
            v = [seeds + _U(P1) + _U(P2), seeds + _U(P2), seeds.copy(), seeds - _U(P1)]
            while p + 32 <= L:
                for k in range(4):
                    v[k] = _vround(v[k], words[:, p // 8 + k])
                p += 32
            h = _vrotl(v[0], 1) + _vrotl(v[1], 7) + _vrotl(v[2], 12) + _vrotl(v[3], 18)
            for k in range(4):
                h = (h ^ _vround(_U(0), v[k])) * _U(P1) + _U(P4)
        else:
            h = seeds + _U(P5)
        h = h + _U(L)
        while p + 8 <= L:
            h = h ^ _vround(_U(0), words[:, p // 8])
            h = _vrotl(h, 27) * _U(P1) + _U(P4)
            p += 8
        if p + 4 <= L:
            w4 = np.ascontiguousarray(mat[:, p:p + 4]).view("<u4").reshape(n).astype(np.uint64)
            h = h ^ (w4 * _U(P1))
            h = _vrotl(h, 23) * _U(P2) + _U(P3)
            p += 4
        while p < L:
            h = h ^ (mat[:, p].astype(np.uint64) * _U(P5))
            h = _vrotl(h, 11) * _U(P1)
            p += 1
        return _vfmix(h)


def _seeds(seed, n):
    if np.isscalar(seed) or isinstance(seed, int):
        return np.full(n, int(seed) & _MASK, dtype=np.uint64)
    return np.asarray(seed, dtype=np.uint64)


def hash_bytes_many(blobs, seed=SEED):
    """XXH64 of every bytes object in `blobs`, grouped by length -> uint64[n]."""
    n = len(blobs)
    seeds = _seeds(seed, n)
    out = np.zeros(n, dtype=np.uint64)
    lens = np.fromiter((len(b) for b in blobs), dtype=np.int64, count=n)
    for L in np.unique(lens).tolist():
        idx = np.nonzero(lens == L)[0]
        mat = np.frombuffer(b"".join(blobs[i] for i in idx.tolist()), dtype=np.uint8).reshape(len(idx), L) \
            if L else np.zeros((len(idx), 0), dtype=np.uint8)
        out[idx] = _xxh64_rows(mat, seeds[idx])
    return out


def typed_words(values, spark_type):
    """Non-NULL values -> (uint8 matrix [n, 4 or 8] of the hashed bytes) for the numeric Spark types."""
    if spark_type in ("int", "boolean"):
        return np.asarray(values, dtype="<i4").reshape(-1, 1).view(np.uint8)
    if spark_type == "long":
        return np.asarray(values, dtype="<i8").reshape(-1, 1).view(np.uint8)
    if spark_type == "float":
        with np.errstate(invalid="ignore"):
            f = np.asarray(values, dtype="<f4").copy()
        f[f == 0] = 0.0
        bits = f.view("<u4").copy()
        bits[np.isnan(f)] = 0x7FC00000
        return bits.reshape(-1, 1).view(np.uint8)
    if spark_type == "double":
        d = np.asarray(values, dtype="<f8").copy()
        d[d == 0] = 0.0
        bits = d.view("<u8").copy()
        bits[np.isnan(d)] = 0x7FF8000000000000
        return bits.reshape(-1, 1).view(np.uint8)
    raise ValueError("unknown Spark type {!r}".format(spark_type))


def hash_values(values, spark_type, seed=SEED):
    """spark_hash over an array of non-NULL values of one Spark type -> uint64[n]."""
    if spark_type == "string":
        return hash_bytes_many([str(v).encode("utf-8") for v in values], seed)
    mat = typed_words(values, spark_type)
    return _xxh64_rows(mat, _seeds(seed, len(mat)))


# ---- registers and the estimate --------------------------------------------------------------------------
def registers(hashes):
    """uint8[512] HLL++ registers of uint64 hashes."""
    h = np.asarray(hashes, dtype=np.uint64)
    regs = np.zeros(M, dtype=np.uint8)
    if len(h) == 0:
        return regs
    idx = (h >> _U(64 - P)).astype(np.int64)
    w = (h << _U(P)) | _U(1 << (P - 1))
    # number of leading zeros of a non-zero uint64: 63 - floor(log2 w), exactly via the bit length of the top half
    hi = (w >> _U(32)).astype(np.int64)
    lo = (w & _U(0xFFFFFFFF)).astype(np.int64)
    nlz = np.where(hi > 0, 32 - _bit_length(hi), 64 - _bit_length(lo))
    np.maximum.at(regs, idx, (nlz + 1).astype(np.uint8))
    return regs


def _bit_length(v):
    v = np.asarray(v, dtype=np.int64)
    out = np.zeros(v.shape, dtype=np.int64)
    for s in (16, 8, 4, 2, 1):
        big = v >= (1 << s)
        out += np.where(big, s, 0)
        v = np.where(big, v >> s, v)
    return out + (v > 0)


def estimate(regs):
    """-> (estimate, in_band): Spark's rounded estimate, or (None, True) when it lies in the bias-table band."""
    regs = np.asarray(regs, dtype=np.int64)
    zeros = int(np.count_nonzero(regs == 0))
    if zeros > 0:
        h = M * math.log(M / zeros)
        if h <= LINEAR_COUNTING_THRESHOLD:
            return _java_round(h), False
    z = float(np.sum(np.ldexp(1.0, -regs)))
    e = ALPHA_M2 / z
    if e >= RAW_ESTIMATE_FLOOR:
        return _java_round(e), False
    return None, True


def _java_round(x):
    return int(math.floor(x + 0.5))


def distinct_count(regs, exact):
    """-> (count, "estimate" | "exact"): the Spark estimate, or `exact` inside the bias-table band."""
    est, band = estimate(regs)
    return (int(exact), "exact") if band else (est, "estimate")


# ---- columns and pairs -----------------------------------------------------------------------------------
def spark_type_of_dtype(dtype):
    """The Spark type a column of this numpy / pandas dtype maps to (IntegerType-like, LongType, ...)."""
    dt = np.dtype(dtype) if not hasattr(dtype, "kind") else dtype
    if dt.kind == "b":
        return "boolean"
    if dt.kind in "iu":
        return "int" if dt.itemsize < 4 or (dt.kind == "i" and dt.itemsize == 4) else "long"
    if dt.kind == "f":
        return "float" if dt.itemsize == 4 else "double"
    return "string"


def column_registers(dictionary, spark_type):
    """Registers of a column with distinct non-NULL values `dictionary`."""
    return registers(hash_values(list(dictionary) if spark_type == "string" else dictionary, spark_type))


def pair_registers(hx, y_values, y_type, present):
    """Registers of struct(x, y) over a presence matrix bool [dom_x + 1, dom_y + 1] (slot 0 = NULL):
    hx[i] = hash of x slot i (hx[0] = 42, a NULL x passes the seed through); y_values: the dom_y values of y."""
    ii, jj = np.nonzero(np.asarray(present, dtype=bool))
    seeds = np.asarray(hx, dtype=np.uint64)[ii]
    out = seeds.copy()
    nn = jj > 0
    if nn.any():
        vals = np.asarray(y_values, dtype=object)[jj[nn] - 1] if y_type == "string" else \
            np.asarray(y_values)[jj[nn] - 1]
        out[nn] = hash_values(vals, y_type, seeds[nn])
    return registers(out)
