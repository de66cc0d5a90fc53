"""``delphi.misc`` (python/repair/misc.py:27-365): the reference's table utilities around a repair.

* ``repair()`` applies a frame of predicted updates ``(row_id, attribute, repaired)`` to an input table
  (RepairMiscApi.scala:184-247);
* ``describe()``, ``toHistogram()``, ``toErrorMap()``, ``injectNull()``, ``flatten()`` and
  ``splitInputTable()`` profile, reshape, perturb and partition a table on the GPU (:41-347).

``generateDepGraph()`` is not provided (it renders through Graphviz).  The utilities take any table from
``repair.catalog`` -- only the row id, when one is given, must exist (RepairBase.scala:101-110); there is no
column-count, uniqueness or type gate.  A registered ``pyarrow.Table`` gives a ``pyarrow.Table`` back from
``flatten``, ``injectNull``, ``toErrorMap`` and ``splitInputTable``; ``describe`` and ``toHistogram`` return
small pandas frames.  Options are validated before any device work; there is no CPU fallback.
"""
import secrets
from typing import Dict, List

import numpy as np
import pandas as pd

from . import catalog
from .table import ROW_ALIGN, encode_columns
from .utils import AnalysisException, argtype_check, cell_to_string, double_to_string, row_positions

_M64 = (1 << 64) - 1
MAX_TARGETS = 64   # columns of one dr_kmeans_assign pass


def _to_double(v):
    """Spark's CAST(string AS DOUBLE): also takes a trailing d/D/f/F type suffix; unparsable -> NULL."""
    if isinstance(v, str):
        v = v.strip()
        if v[-1:] in "dDfF" and v[:-1]:
            v = v[:-1]
    try:
        return float(v)
    except (TypeError, ValueError):
        return float("nan")


class RepairMisc():

    def __init__(self) -> None:
        self.opts: Dict[str, str] = {}

    @argtype_check
    def option(self, key: str, value: str) -> "RepairMisc":
        self.opts[str(key)] = str(value)
        return self

    @argtype_check
    def options(self, options: Dict[str, str]) -> "RepairMisc":
        self.opts.update(options)
        return self

    def _check_required_options(self, required: List[str]) -> None:
        if not all(opt in self.opts.keys() for opt in required):
            raise ValueError("Required options not found: {}".format(", ".join(required)))

    # ---- option helpers (python/repair/misc.py:60-85) --------------------------------------------------
    @property
    def _db_name(self) -> str:
        return self.opts.get("db_name", "")

    @property
    def _target_attr_list(self) -> str:
        return self.opts.get("target_attr_list", "")

    def _load(self, row_id=""):
        """checkAndGetQualifiedInputName (RepairBase.scala:101-110) -> (table, qualified name, column names)."""
        name = "{}.{}".format(self._db_name, self.opts["table_name"]) if self._db_name else self.opts["table_name"]
        tbl = catalog.table(name)
        columns = [str(c) for c in (tbl.columns if isinstance(tbl, pd.DataFrame) else tbl.column_names)]
        if row_id and row_id not in columns:
            raise AnalysisException("Column '{}' does not exist in '{}'.".format(row_id, name))
        return tbl, name, columns

    @staticmethod
    def _attr_list(value, columns, name):
        attrs = _to_seq(value)
        unknown = [a for a in attrs if a not in columns]
        if unknown:
            raise AnalysisException("Columns '{}' do not exist in '{}'".format(", ".join(unknown), name))
        return attrs

    def repair(self) -> pd.DataFrame:
        """Applies predicted repair updates into an input table: a cell whose (row id, attribute) is
        listed takes the `repaired` value -- cast to the column's type, rounded first for integral
        columns (RepairMiscApi.scala:224-230) -- every other cell is kept; when a cell is listed twice
        the last update wins (Spark's map_from_entries keeps the last duplicate key under
        spark.sql.mapKeyDedupPolicy=LAST_WIN; the default policy raises instead)."""
        self._check_required_options(["repair_updates", "table_name", "row_id"])
        row_id = self.opts["row_id"]
        name = self.opts["table_name"]
        if self.opts.get("db_name"):
            name = "{}.{}".format(self.opts["db_name"], name)
        table = catalog.table(name)
        updates = catalog.table(self.opts["repair_updates"])
        if not all(c in updates.columns for c in (row_id, "attribute", "repaired")):
            raise AnalysisException("Table '{}' must have '{}', 'attribute', and 'repaired' columns".format(
                self.opts["repair_updates"], row_id))
        out = table.copy()
        ids = out[row_id].to_numpy()
        for attr, grp in updates.groupby("attribute", sort=False):
            if attr not in out.columns or attr == row_id:
                continue
            col = out[attr]
            # vectorised join on the row id (no Python dict over the table's rows)
            pos, found = row_positions(ids, grp[row_id].to_numpy())
            rows = pos[found].tolist()
            vals = [None if v is None or (isinstance(v, float) and v != v) else v
                    for v, f in zip(grp["repaired"].tolist(), found.tolist()) if f]
            if not rows:
                continue
            if pd.api.types.is_integer_dtype(col.dtype):
                arr = col.astype("Int64").to_numpy(dtype=object, copy=True)
                for i, v in zip(rows, vals):
                    d = np.nan if v is None else _to_double(v)
                    # Spark's round() is half-up (away from zero), unlike numpy's half-even
                    arr[i] = pd.NA if d != d else int(np.floor(abs(d) + 0.5) * (1 if d >= 0 else -1))
                out[attr] = pd.array(arr, dtype="Int64")
            elif pd.api.types.is_float_dtype(col.dtype):
                arr = col.to_numpy(dtype=np.float64, copy=True)
                for i, v in zip(rows, vals):
                    arr[i] = np.nan if v is None else _to_double(v)
                out[attr] = arr
            else:
                arr = col.to_numpy(dtype=object, copy=True)
                for i, v in zip(rows, vals):
                    arr[i] = v
                out[attr] = arr
        return out

    # ---- profiling -----------------------------------------------------------------------------------
    def describe(self) -> pd.DataFrame:
        """Column stats (computeAndGetStats, RepairMiscApi.scala:249-275): one row per column in schema order
        with ``attrName, distinctCnt, min, max, nullCnt, avgLen, maxLen, hist``.  ``min`` / ``max`` are the
        CAST(.. AS STRING) of numeric extremes; ``avgLen`` / ``maxLen`` are the ceiling of the mean and the
        maximum character length of strings (20, Spark's defaultSize, for an all-NULL string column) and the
        source type's size for numbers; ``hist`` (numbers only) are the gaps between the percentiles at
        i / num_bins (the ceil(p n)-th smallest value) normalised by their sum.  One dr_scan_hist pass.
        Option ``spark_compatible_distinct_counts`` ("true" / "false", default "false"): ``distinctCnt`` is
        Spark's HyperLogLog++ estimate (repair/hll.py; the exact count inside the bias-table band)."""
        self._check_required_options(["table_name"])
        spark_ndv = self.opts.get("spark_compatible_distinct_counts", "false").strip().lower()
        if spark_ndv not in ("true", "false"):
            raise ValueError("Option 'spark_compatible_distinct_counts' must be 'true' or 'false', but '{}' "
                             "found".format(self.opts["spark_compatible_distinct_counts"]))
        num_bins = 8
        if "num_bins" in self.opts:
            try:
                num_bins = int(self.opts["num_bins"])
            except ValueError:
                raise ValueError("Option 'num_bins' must be an integer, but '{}' found".format(
                    self.opts["num_bins"])) from None
            if num_bins < 2:      # spark.sql.statistics.histogram.numBins' own check
                raise ValueError("The number of bins must be greater than 1, but {} found".format(num_bins))
        tbl, _, _ = self._load()
        cols = encode_columns(tbl)
        hists = _device_hists(cols)
        ndv = {}
        if spark_ndv == "true":
            from . import hll as HLL
            ctx, device = _acquire()
            try:
                ndv = HLL.column_counts(ctx, device, cols)
            finally:
                _release(ctx)
        rows = []
        for col, h in zip(cols, hists):
            cnt = h[1:]
            present = np.nonzero(cnt)[0]
            mn = mx = hist = None
            if col.continuous:
                avg_len = max_len = col.default_size
                if len(present):
                    mn = cell_to_string(col.kind, float(col.dictionary[present[0]]))
                    mx = cell_to_string(col.kind, float(col.dictionary[present[-1]]))
                    hist = percentile_hist(np.asarray(col.dictionary, dtype=np.float64), cnt, num_bins)
            else:
                n = int(cnt.sum())
                if n:
                    lens = np.array([len(s) for s in col.strings()], dtype=np.int64)
                    avg_len = -(-int((lens * cnt).sum()) // n)
                    max_len = int(lens[present].max())
                else:
                    avg_len = max_len = col.default_size
            distinct = ndv[col.name][0] if ndv else int(len(present))
            rows.append((col.name, distinct, mn, mx, int(h[0]), int(avg_len), int(max_len), hist))
        names = ["attrName", "distinctCnt", "min", "max", "nullCnt", "avgLen", "maxLen", "hist"]
        return pd.DataFrame({c: pd.Series([r[i] for r in rows], dtype=object if c in ("attrName", "min", "max", "hist")
                                           else np.int64) for i, c in enumerate(names)})

    def toHistogram(self) -> pd.DataFrame:
        """Value counts of the listed string columns (convertToHistogram, RepairMiscApi.scala:277-302):
        ``attribute, histogram`` with ``histogram`` a list of ``{"value", "cnt"}`` of the non-NULL values;
        numeric columns and unknown names are skipped.  One dr_scan_hist pass."""
        self._check_required_options(["table_name", "targets"])
        tbl, _, columns = self._load()
        targets = set(_to_seq(self.opts["targets"]))
        picked = [c for c in columns if c in targets]
        cols = [c for c in encode_columns(_select(tbl, picked)) if not c.continuous] if picked else []
        hists = _device_hists(cols) if cols else []
        rows = [(c.name, [{"value": s, "cnt": int(n)} for s, n in zip(c.strings(), h[1:].tolist()) if n])
                for c, h in zip(cols, hists)]
        return pd.DataFrame(rows, columns=["attribute", "histogram"])

    # ---- reshaping -----------------------------------------------------------------------------------
    def toErrorMap(self):
        """One ``*`` (error) or ``-`` per non-row-id column, in schema order, for every row (toErrorMap,
        RepairMiscApi.scala:304-347): ``row_id, error_map``.  Error cells whose row id or attribute is not in
        the table are ignored.  The characters are written by dr_error_map from per-attribute bitmaps."""
        self._check_required_options(["table_name", "row_id", "error_cells"])
        row_id = self.opts["row_id"]
        cells = catalog.table(self.opts["error_cells"])
        cell_cols = cells.columns if isinstance(cells, pd.DataFrame) else cells.column_names
        if row_id not in cell_cols or "attribute" not in cell_cols:
            raise AnalysisException("Table '{}' must have '{}' and 'attribute' columns".format(
                self.opts["error_cells"], row_id))
        tbl, _, columns = self._load(row_id)
        if not isinstance(cells, pd.DataFrame):
            cells = cells.select([row_id, "attribute"]).to_pandas()
        attrs = [c for c in columns if c != row_id]
        ids = _column_numpy(tbl, row_id)
        n, K = len(ids), len(attrs)
        if K == 0 or n == 0:
            chars = np.zeros(n * K, dtype=np.uint8)
        else:
            import torch
            ctx, device = _acquire()
            try:
                words = (n + 31) // 32
                maps = [None] * K
                index = {a: i for i, a in enumerate(attrs)}
                for attr, grp in cells.groupby("attribute", sort=False):
                    if attr not in index:
                        continue
                    pos, found = row_positions(ids, grp[row_id].to_numpy())
                    pos = pos[found]
                    bits = np.zeros(words, dtype=np.uint32)
                    np.bitwise_or.at(bits, pos >> 5, (np.uint32(1) << (pos & 31).astype(np.uint32)))
                    maps[index[attr]] = torch.from_numpy(bits.view(np.int32)).to(device)
                out = torch.empty(n * K, dtype=torch.uint8, device=device)
                ctx.error_map(maps, n, out)
                chars = out.cpu().numpy()
            finally:
                _release(ctx)
        if isinstance(tbl, pd.DataFrame):
            strs = chars.view("S{}".format(K)).astype("U{}".format(K)).astype(object) if K else \
                np.full(n, "", dtype=object)
            return pd.DataFrame({row_id: tbl[row_id].to_numpy(), "error_map": strs})
        import pyarrow as pa
        offs = np.arange(n + 1, dtype=np.int64) * K
        if offs[-1] < 2 ** 31:
            arr = pa.StringArray.from_buffers(n, pa.py_buffer(offs.astype(np.int32)), pa.py_buffer(chars))
        else:
            arr = pa.LargeStringArray.from_buffers(n, pa.py_buffer(offs), pa.py_buffer(chars))
        return pa.table({row_id: tbl[row_id], "error_map": arr})

    def flatten(self):
        """``row_id, attribute, value`` with ``value = CAST(.. AS STRING)``, row-major, attributes in schema
        order (flattenTable, RepairMiscApi.scala:41-49).  dr_flatten writes every cell's code in one
        concatenated dictionary, its validity and the repeated row id; Arrow output is three Arrow arrays
        (attribute and value dictionary-encoded) without a Python object per cell."""
        self._check_required_options(["table_name", "row_id"])
        row_id = self.opts["row_id"]
        tbl, _, columns = self._load(row_id)
        attrs = [c for c in columns if c != row_id]
        ids = _column_numpy(tbl, row_id)
        n, K = len(ids), len(attrs)
        cols = encode_columns(_select(tbl, attrs)) if attrs else []
        strings = [c.strings() for c in cols]
        base = np.concatenate([[0], np.cumsum([len(s) for s in strings])]).astype(np.int64)
        values = [v for s in strings for v in s]
        int_ids = ids.dtype.kind in "iu"
        total = n * K
        if total == 0:
            codes = np.zeros(0, dtype=np.int32)
            valid = np.zeros(0, dtype=bool)
            out_ids = np.zeros(0, dtype=np.int64)
        else:
            import torch
            ctx, device = _acquire()
            try:
                d_codes = _upload_codes(cols, n, device)
                d_ids = torch.from_numpy(ids.astype(np.int64)).to(device) if int_ids else None
                o_codes = torch.empty(total, dtype=torch.int32, device=device)
                o_valid = torch.empty((total + 31) // 32, dtype=torch.int32, device=device)
                o_ids = torch.empty(total, dtype=torch.int64, device=device)
                ctx.flatten(list(d_codes), base[:-1], n, d_ids, o_codes, o_valid, o_ids)
                codes, out_ids = o_codes.cpu().numpy(), o_ids.cpu().numpy()
                vbits = o_valid.cpu().numpy()
            finally:
                _release(ctx)
            valid = np.unpackbits(vbits.view(np.uint8), bitorder="little")[:total].astype(bool)
        attr_idx = np.tile(np.arange(K, dtype=np.int32), n)
        if isinstance(tbl, pd.DataFrame):
            rid = out_ids.astype(ids.dtype) if int_ids else ids[out_ids]
            vals = np.array(values + [None], dtype=object)[np.where(valid, codes, len(values))] if total else \
                np.zeros(0, dtype=object)
            return pd.DataFrame({row_id: rid, "attribute": np.array(attrs, dtype=object)[attr_idx], "value": vals})
        import pyarrow as pa
        id_col = tbl[row_id].combine_chunks() if tbl[row_id].num_chunks != 1 else tbl[row_id].chunk(0)
        rid = pa.array(out_ids).cast(id_col.type) if int_ids else id_col.take(pa.array(out_ids))
        vbuf = pa.py_buffer(vbits) if total else None
        idx = pa.Array.from_buffers(pa.int32(), total, [vbuf, pa.py_buffer(codes)])
        value = pa.DictionaryArray.from_arrays(idx, pa.array(values, type=pa.string()))
        attribute = pa.DictionaryArray.from_arrays(pa.array(attr_idx), pa.array(attrs, type=pa.string()))
        return pa.table({row_id: rid, "attribute": attribute, "value": value})

    # ---- benchmark construction ----------------------------------------------------------------------
    def injectNull(self, _seed=None):
        """``IF(rand() > null_ratio, x, NULL)`` on every cell of the listed columns, every column when the
        list is empty (injectNullAt, RepairMiscApi.scala:155-182).  rand() is splitmix64 over (seed, column,
        row) -- the hash of ``repair.synth`` -- evaluated by dr_null_bits, which writes new validity bitmaps:
        Arrow columns keep their values buffers and only change validity.  Like Spark's unseeded rand(),
        each call draws a fresh seed."""
        self._check_required_options(["table_name", "target_attr_list"])
        if "null_ratio" in self.opts:
            try:
                ratio = float(self.opts["null_ratio"])
                ok = 0.0 < ratio <= 1.0
            except ValueError:
                ok = False
            if not ok:
                raise ValueError("Option 'null_ratio' must be a float in (0.0, 1.0], "
                                 "but '{}' found".format(self.opts["null_ratio"]))
        else:
            ratio = 0.01
        tbl, name, columns = self._load()
        targets = set(self._attr_list(self._target_attr_list, columns, name)) or set(columns)
        seed = secrets.randbits(63) if _seed is None else int(_seed)
        import torch
        ctx, device = _acquire()
        try:
            if isinstance(tbl, pd.DataFrame):
                out = tbl.copy()
                n = len(tbl)
                for ci, c in enumerate(columns):
                    if c not in targets or n == 0:
                        continue
                    s = tbl[tbl.columns[ci]]
                    valid = np.packbits(~pd.isna(s).to_numpy(), bitorder="little")
                    keep = _null_bits(ctx, device, torch, valid, 0, n, 0, null_key(seed, ci), ratio)
                    out[out.columns[ci]] = _mask_series(s, keep)
                return out
            import pyarrow as pa
            arrays = []
            for ci, c in enumerate(columns):
                col = tbl.column(ci)
                if c not in targets or pa.types.is_null(col.type):
                    arrays.append(col)
                    continue
                chunks, row_base = [], 0
                for ch in col.chunks:
                    chunks.append(_arrow_null_chunk(ctx, device, torch, ch, row_base, null_key(seed, ci), ratio))
                    row_base += len(ch)
                arrays.append(pa.chunked_array(chunks, type=col.type))
            return pa.Table.from_arrays(arrays, schema=tbl.schema)
        finally:
            _release(ctx)

    def splitInputTable(self):
        """Splits the rows into k groups of similar rows (splitInputTableInto, RepairMiscApi.scala:75-153):
        ``row_id, k``.  A row's features are the bag of q-grams of its target cells' CAST(.. AS STRING)
        values (NULL cells skipped).  As in the reference the algorithm names are crossed:
        ``clustering_alg="bisect-kmeans"`` (the default) runs k-means and ``"kmeans++"`` runs bisecting
        k-means.  The clustering runs on dictionary codes (``repair.cluster``): each iteration is one
        dr_kmeans_assign pass and one dr_cooc pass over the table."""
        self._check_required_options(["table_name", "row_id", "k"])
        if not self.opts["k"].isdigit():
            raise ValueError("Option 'k' must be an integer, but '{}' found".format(self.opts["k"]))
        k = int(self.opts["k"])
        q_opt = self.opts.get("q", "2")
        alg = self.opts.get("clustering_alg", "bisect-kmeans")
        row_id = self.opts["row_id"]
        tbl, name, columns = self._load(row_id)
        targets = self._attr_list(self._target_attr_list, columns, name) or [c for c in columns if c != row_id]
        try:
            q = int(q_opt)
        except ValueError:
            q = 2
        if alg not in ("bisect-kmeans", "kmeans++"):
            raise ValueError("Unknown clustering algorithm found: {}".format(alg))
        if len(targets) > MAX_TARGETS:
            raise ValueError("splitInputTable takes at most {} target columns, but {} found: list the columns to "
                             "cluster on in 'target_attr_list'".format(MAX_TARGETS, len(targets)))
        if k < 2:
            raise ValueError("k must be greater than 1, but {} found".format(k))
        if q <= 0:
            raise ValueError("`q` must be positive, but {} got".format(q))
        labels = split_table(tbl, targets, k, q, alg)
        if isinstance(tbl, pd.DataFrame):
            return pd.DataFrame({row_id: tbl[row_id].to_numpy(), "k": labels})
        import pyarrow as pa
        return pa.table({row_id: tbl[row_id], "k": pa.array(labels, type=pa.int32())})


# ---- helpers -------------------------------------------------------------------------------------------
def _to_seq(s):
    """SparkUtils.stringToSeq: comma-separated, trimmed, empty entries dropped."""
    return [t.strip() for t in str(s).split(",") if t.strip()]


def _select(tbl, names):
    return tbl[names] if isinstance(tbl, pd.DataFrame) else tbl.select(names)


def _column_numpy(tbl, name):
    if isinstance(tbl, pd.DataFrame):
        return tbl[name].to_numpy()
    return np.asarray(tbl[name].to_numpy())


def _acquire():
    import torch
    from ._native import Context, NativeError
    if not torch.cuda.is_available():
        raise NativeError("no CUDA device is available; delphi.misc has no CPU fallback")
    index = torch.cuda.current_device()
    return Context.acquire(index), torch.device("cuda", index)


def _release(ctx):
    from ._native import Context
    Context.release(ctx)


def _upload_codes(cols, n, device):
    """int32 [K][n_pad] device codes (NULL and padding = -1), every column 512-byte aligned."""
    import torch
    n_pad = (n + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN or ROW_ALIGN
    host = np.full((len(cols), n_pad), -1, dtype=np.int32)
    for i, c in enumerate(cols):
        host[i, :n] = c.codes
    return torch.from_numpy(host).to(device)


def _device_hists(cols, ctx=None, device=None, codes=None):
    """Slot counts of every column (slot 0 = NULL, slot v + 1 = dictionary entry v) from one dr_scan_hist."""
    import torch
    if not cols:
        return []
    n = len(cols[0].codes)
    own = ctx is None
    if own:
        ctx, device = _acquire()
    try:
        if codes is None:
            codes = _upload_codes(cols, n, device)
        dom = [c.dict_size for c in cols]
        off = np.concatenate([[0], np.cumsum([d + 1 for d in dom])]).astype(np.int64)
        hist = torch.zeros(int(off[-1]), dtype=torch.int64, device=device)
        for c0 in range(0, len(cols), 64):
            part = list(range(c0, min(len(cols), c0 + 64)))
            ctx.scan_hist([codes[i] for i in part], [dom[i] for i in part], n, [None] * len(part),
                          hist[int(off[c0]):])
        h = hist.cpu().numpy()
    finally:
        if own:
            _release(ctx)
    return [h[off[i]:off[i + 1]] for i in range(len(cols))]


def percentile_hist(values, cnt, num_bins):
    """Gaps between the percentiles at i / num_bins (the ceil(p n)-th smallest value, the smallest for p = 0)
    normalised by their sum (RepairMiscApi.scala:256-260); values sorted, cnt their multiplicities."""
    cnt = np.asarray(cnt, dtype=np.int64)
    n = int(cnt.sum())
    cum = np.cumsum(cnt)
    ranks = np.array([max(1, -(-i * n // num_bins)) for i in range(num_bins + 1)], dtype=np.int64)
    pct = np.asarray(values, dtype=np.float64)[np.searchsorted(cum, ranks, side="left")]
    gaps = np.diff(pct)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (gaps / gaps.sum()).tolist()


def null_key(seed, col):
    """The additive key of ``repair.synth._mix_np(seed, col, rows)``."""
    return (int(seed) * 0x2545F4914F6CDD1D + (int(col) + 1) * 0xD6E8FEB86659FD93) & _M64


def _null_bits(ctx, device, torch, valid_bytes, bit_offset, n, row_base, key, ratio):
    """valid_bytes (uint8 bitmap or None) -> kept bits as a uint8 bitmap of ceil((bit_offset + n) / 32) words."""
    words = (bit_offset + n + 31) // 32
    d_valid = None
    if valid_bytes is not None:
        buf = np.zeros(words * 4, dtype=np.uint8)
        m = min(len(valid_bytes), words * 4)
        buf[:m] = valid_bytes[:m]
        d_valid = torch.from_numpy(buf.view(np.int32)).to(device)
    out = torch.empty(words, dtype=torch.int32, device=device)
    ctx.null_bits(d_valid, bit_offset, n, row_base, key, ratio, out)
    return out.cpu().numpy().view(np.uint8)


def _mask_series(s, keep_bits):
    keep = np.unpackbits(keep_bits, bitorder="little")[:len(s)].astype(bool)
    if s.dtype.kind in "iu" and isinstance(s.dtype, np.dtype):
        return pd.Series(pd.arrays.IntegerArray(s.to_numpy(), ~keep), index=s.index, name=s.name)
    if s.dtype.kind == "b" and isinstance(s.dtype, np.dtype):
        return pd.Series(pd.arrays.BooleanArray(s.to_numpy(), ~keep), index=s.index, name=s.name)
    return s.where(keep, None) if s.dtype == object else s.where(keep)


def _arrow_null_chunk(ctx, device, torch, arr, row_base, key, ratio):
    """New validity bitmap for one Arrow chunk (same bit offset); the values buffers are reused."""
    import pyarrow as pa
    n = len(arr)
    if n == 0:
        return arr
    target = arr.indices if pa.types.is_dictionary(arr.type) else arr
    bufs = target.buffers()
    off = target.offset
    valid = None if bufs[0] is None else np.frombuffer(bufs[0], dtype=np.uint8)
    bits = _null_bits(ctx, device, torch, valid, off, n, row_base, key, ratio)
    new = pa.Array.from_buffers(target.type, n, [pa.py_buffer(bits)] + bufs[1:], offset=off)
    if pa.types.is_dictionary(arr.type):
        return pa.DictionaryArray.from_arrays(new, arr.dictionary)
    return new


def target_strings(cols):
    """CAST(.. AS STRING) of the dictionary entries of splitInputTable's target columns as elements of the
    reference's ``array(targets)``: Spark coerces the array to one element type, so when every target is numeric
    and one of them is floating, integer cells print as doubles ("1.0"); any string target keeps every column's
    own text."""
    as_double = all(c.continuous for c in cols) and any(c.kind == "float" for c in cols)
    return [[double_to_string(float(v)) for v in c.dictionary] if as_double and c.kind == "int" else c.strings()
            for c in cols]


def split_table(tbl, targets, k, q, alg, info=None):
    """Labels 0..k-1 (int32, one per row) of splitInputTable on the listed columns; see ``repair.cluster``."""
    from . import cluster
    names = list(dict.fromkeys(targets))
    cols = encode_columns(_select(tbl, names))
    by_name = {c.name: c for c in cols}
    order = [by_name[t] for t in targets]
    n = len(tbl)
    if n == 0:
        return np.zeros(0, dtype=np.int32)
    ctx, device = _acquire()
    try:
        codes = _upload_codes(cols, n, device)
        dev = {c.name: codes[i] for i, c in enumerate(cols)}
        hists = dict(zip(names, _device_hists(cols, ctx, device, codes)))
        hist = [hists[t] for t in targets]
        feats = cluster.QgramFeatures(target_strings(order), hist, q)
        dk = cluster.DeviceKMeans(ctx, [dev[t] for t in targets], feats, n, device)
        if alg == "bisect-kmeans":          # the reference's crossed names: this one is k-means
            labels = cluster.kmeans(dk, k, info).cpu().numpy()[:n]
        else:
            lab, lut = cluster.bisecting_kmeans(dk, k, hist, n, info)
            labels = lut[lab.cpu().numpy()[:n]]
    finally:
        _release(ctx)
    return labels.astype(np.int32)
