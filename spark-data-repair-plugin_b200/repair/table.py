"""Host-side table ingest: a DataFrame is collected ONCE into label-encoded int32 column-major
arrays (sorted dictionaries, NULL = -1) plus float64 side arrays for numeric columns, then copied
to the GPU through pinned staging buffers.  This replaces the Spark views the reference passes by
name between Python and Scala (SURVEY.md section 8b, "Data hand-off").
"""
import numpy as np

from .utils import AnalysisException, cell_to_string

_SUPPORTED_MSG = "tinyint,float,smallint,string,double,int,bigint"  # RepairBase.scala:41-44 order as Spark prints it
INGEST_GROUP_COLS = 8   # Arrow columns per copy / encode group of the device-side ingest
ROW_ALIGN = 128  # rows are padded so that every column starts 512-byte aligned (128-bit loads)


class Column:
    """kind: 'str' (discrete) | 'int' | 'float' (both continuous, RepairBase.scala:41-44).
    ``dictionary``: sorted distinct non-NULL values (str objects, or float64 for numerics);
    ``codes``: int32 index into it, -1 = NULL;  ``values``: float64 (NaN = NULL) for numerics.
    ``spark_type``: the Spark type of the source column ('string', 'int', 'long', 'float', 'double',
    'boolean'), or None when unknown; only the Spark-compatible distinct counts (repair/hll.py) read it."""

    def __init__(self, name, kind, dictionary, codes, values=None, spark_type=None):
        self.name, self.kind, self.dictionary, self.values = name, kind, dictionary, values
        self.spark_type = spark_type
        self._codes = codes      # host int32 array, or a callable that fetches it (device-resident ingest)

    @property
    def codes(self):
        if callable(self._codes):
            self._codes = self._codes()
        return self._codes

    @codes.setter
    def codes(self, v):
        self._codes = v

    @property
    def dict_size(self):
        return len(self.dictionary)

    @property
    def continuous(self):
        return self.kind in ("int", "float")

    def code_of(self, value):
        """Dictionary code of a python value, or -2 if it does not occur."""
        if len(self.dictionary) == 0:
            return -2
        if self.kind == "str":
            if getattr(self, "_lut", None) is None:
                self._lut = {str(v): i for i, v in enumerate(self.dictionary)}
            return self._lut.get(str(value), -2)
        try:
            x = float(value)
        except (TypeError, ValueError):
            return -2
        i = int(np.searchsorted(self.dictionary, x))
        return i if i < len(self.dictionary) and self.dictionary[i] == x else -2

    def rank_bounds(self, value):
        """(lower_bound, upper_bound) ranks of a constant in the sorted dictionary: ``col < c`` is
        ``code < lower`` and ``col > c`` is ``code >= upper``."""
        if self.kind == "str":
            keys = [str(v) for v in self.dictionary]
            import bisect
            return bisect.bisect_left(keys, str(value)), bisect.bisect_right(keys, str(value))
        x = float(value)
        return int(np.searchsorted(self.dictionary, x, "left")), int(np.searchsorted(self.dictionary, x, "right"))

    def strings(self):
        """CAST(dictionary entry AS STRING) for every entry (regex LUTs, output frames)."""
        if self.kind == "str":
            return [str(v) for v in self.dictionary]
        return [cell_to_string(self.kind, float(v)) for v in self.dictionary]

    def decode(self, codes):
        """codes -> list of CAST(.. AS STRING) python values (None for NULL)."""
        strs = self.strings()
        return [None if c < 0 else strs[c] for c in np.asarray(codes).tolist()]


def _encode_numeric(name, kind, arr, spark_type=None):
    vals = np.asarray(arr, dtype=np.float64)
    nul = np.isnan(vals)
    uniq = np.unique(vals[~nul])
    codes = np.full(len(vals), -1, dtype=np.int32)
    codes[~nul] = np.searchsorted(uniq, vals[~nul]).astype(np.int32)
    return Column(name, kind, uniq, codes, vals, spark_type)


def _numpy_spark_type(dtype, kind):
    """Spark type of a numeric numpy / pandas dtype (int8 / int16 / int32 -> int, int64 -> long, float32 -> float,
    float64 -> double); columns of Python objects take the widest type of their kind."""
    k, size = getattr(dtype, "kind", "O"), int(getattr(dtype, "itemsize", 8))
    if k in "iu":
        return "int" if size < 4 or (k == "i" and size == 4) else "long"
    if k == "f":
        return "float" if size <= 4 else "double"
    return "long" if kind == "int" else "double"


def _arrow_spark_type(t):
    import pyarrow as pa
    if pa.types.is_boolean(t):
        return "boolean"
    if pa.types.is_integer(t):
        return "int" if t.bit_width < 32 or (t.bit_width == 32 and pa.types.is_signed_integer(t)) else "long"
    if pa.types.is_floating(t):
        return "float" if t.bit_width <= 32 else "double"
    return "string"


def _encode_arrow_strings(name, arr):
    """pyarrow string / dictionary<string> array (one chunk) -> Column: Arrow's C++ dictionary_encode, then only
    the dictionary (one entry per distinct value) is sorted and turned into Python strings."""
    import pyarrow as pa
    import pyarrow.compute as pc
    if not pa.types.is_dictionary(arr.type):
        arr = pc.dictionary_encode(arr)
    idx = arr.indices
    valid = np.asarray(idx.is_valid())
    raw = np.asarray(idx.fill_null(0).to_numpy(zero_copy_only=False), dtype=np.int64)
    entries = arr.dictionary.to_pylist()
    # a Parquet dictionary page may list values the rows never use: keep what occurs, sorted
    used = np.zeros(len(entries), dtype=bool)
    used[raw[valid]] = True
    dictionary, lut = _sorted_dictionary(entries, used)
    codes = np.where(valid, lut[raw], -1).astype(np.int32) if len(entries) else np.full(len(raw), -1, dtype=np.int32)
    return Column(name, "str", dictionary, codes, None, "string")


def _encode_strings(name, series):
    import pandas as pd
    if series.dtype == object or str(series.dtype) in ("string", "str"):
        # all-string columns (the usual case) never become one Python object per cell: Arrow encodes them;
        # anything else (mixed objects that need str()) takes the generic path below
        try:
            import pyarrow as pa
            arr = pa.array(series.to_numpy(dtype=object, na_value=None) if series.dtype != object else series.to_numpy(),
                           type=pa.string(), from_pandas=True)
            return _encode_arrow_strings(name, arr)
        except Exception:  # noqa: BLE001  (non-string objects, no pyarrow)
            pass
    obj = series.astype(object)
    isn = pd.isna(obj).to_numpy()
    strs = np.array([None if n else str(v) for v, n in zip(obj.tolist(), isn.tolist())], dtype=object)
    present = strs[~isn]
    uniq = np.array(sorted(set(present.tolist())), dtype=object)
    lut = {v: i for i, v in enumerate(uniq.tolist())}
    codes = np.full(len(strs), -1, dtype=np.int32)
    if len(present):
        codes[~isn] = np.fromiter((lut[v] for v in present.tolist()), dtype=np.int32, count=len(present))
    return Column(name, "str", uniq, codes, None, "string")


def _arrow_gate(tbl, row_id, name):
    """checkInputTable's schema gate (RepairApi.scala:34-52) on a pyarrow schema -> {column: kind}."""
    import pyarrow as pa
    if row_id not in tbl.column_names:
        raise AnalysisException("Column '{}' does not exist in table '{}'".format(row_id, name))
    kinds, bad = {}, []
    for f in tbl.schema:
        t = f.type.value_type if pa.types.is_dictionary(f.type) else f.type
        if pa.types.is_boolean(t):
            bad.append("boolean")
        elif pa.types.is_integer(t):
            kinds[f.name] = "int"
        elif pa.types.is_floating(t):
            kinds[f.name] = "float"
        elif pa.types.is_string(t) or pa.types.is_large_string(t):
            kinds[f.name] = "str"
        elif pa.types.is_timestamp(t):
            bad.append("timestamp")
        elif pa.types.is_date(t):
            bad.append("date")
        else:
            bad.append(str(t))
    if bad:
        raise AnalysisException("Supported types are {}, but unsupported ones found: {}".format(
            _SUPPORTED_MSG, ",".join(bad)))
    if not tbl.num_columns >= 3:
        raise AnalysisException("A least three columns (`{}` columns + two more ones) in table '{}'".format(
            row_id, name))
    return kinds


def _sorted_dictionary(entries, used):
    """Arrow dictionary entries + which of them occur -> (sorted dictionary of the occurring non-null
    entries as str objects, int32 LUT old index -> code in it or -1)."""
    used = np.asarray(used, dtype=bool) & np.array([e is not None for e in entries], dtype=bool) \
        if len(entries) else np.zeros(0, dtype=bool)
    keep = np.nonzero(used)[0]
    strs = [str(entries[i]) for i in keep]
    order = keep[np.argsort(np.array(strs, dtype=object), kind="stable")] if len(keep) else keep
    # two dictionary entries may print alike (never for strings; kept for safety): first one wins the code
    uniq, lut = [], np.full(len(entries), -1, dtype=np.int32)
    for i in order:
        v = str(entries[i])
        if not uniq or uniq[-1] != v:
            uniq.append(v)
        lut[i] = len(uniq) - 1
    return np.array(uniq, dtype=object), lut


STRING_DEFAULT_SIZE = 20   # Spark's StringType.defaultSize


def encode_columns(tbl):
    """Every column of a ``pandas.DataFrame`` or ``pyarrow.Table`` label-encoded in schema order, with none of
    checkInputTable's gates: the delphi.misc utilities take any table (RepairBase.scala:101-110).  Integer and
    floating columns are numeric; everything else is encoded by its ``CAST(.. AS STRING)`` text.  Each Column
    also carries ``default_size``: Spark's defaultSize of the source type (tinyint 1, smallint 2, int 4,
    bigint 8, float 4, double 8; strings 20), which ``describe`` reports for numeric columns."""
    import pandas as pd
    cols = []
    if isinstance(tbl, pd.DataFrame):
        for c in tbl.columns:
            s = tbl[c]
            k = s.dtype.kind
            kind = "int" if k in "iu" else "float" if k == "f" else None
            size = int(getattr(s.dtype, "itemsize", 8)) if kind else 8
            if kind is None and s.dtype == object:
                # object columns holding only numbers (e.g. nullable ints collected from Spark) are numeric
                non_null = [v for v in s.tolist() if v is not None and not (isinstance(v, float) and v != v)]
                if non_null and all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in non_null):
                    kind = "int"
                elif non_null and all(isinstance(v, (int, float, np.integer, np.floating)) and
                                      not isinstance(v, bool) for v in non_null):
                    kind = "float"
            if kind is not None:
                arr = pd.to_numeric(s, errors="coerce").to_numpy(dtype=np.float64, na_value=np.nan)
                col = _encode_numeric(str(c), kind, arr, _numpy_spark_type(s.dtype, kind))
            else:
                if k == "b":
                    s = s.map(lambda v: None if v is None or v != v else ("true" if v else "false"))
                col = _encode_strings(str(c), s)
                if k == "b":
                    col.spark_type = "boolean"
                size = STRING_DEFAULT_SIZE
            col.default_size = size
            cols.append(col)
        return cols
    import pyarrow as pa
    import pyarrow.compute as pc
    for f in tbl.schema:
        arr = tbl[f.name]
        arr = arr.unify_dictionaries() if pa.types.is_dictionary(f.type) else arr
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
        t = f.type.value_type if pa.types.is_dictionary(f.type) else f.type
        if pa.types.is_integer(t) or pa.types.is_floating(t):
            if pa.types.is_dictionary(arr.type):
                arr = arr.dictionary_decode()
            vals = np.asarray(pc.cast(arr, pa.float64()).to_numpy(zero_copy_only=False), dtype=np.float64)
            col = _encode_numeric(f.name, "int" if pa.types.is_integer(t) else "float", vals, _arrow_spark_type(t))
            col.default_size = t.bit_width // 8
        else:
            if not (pa.types.is_string(t) or pa.types.is_large_string(t)):
                arr = pc.cast(arr.dictionary_decode() if pa.types.is_dictionary(arr.type) else arr, pa.string())
            col = _encode_arrow_strings(f.name, arr)
            col.spark_type = _arrow_spark_type(t)
            col.default_size = STRING_DEFAULT_SIZE
        cols.append(col)
    return cols


class EncodedTable:
    """The collected input: row ids + encoded columns (row id excluded)."""

    def __init__(self, row_id, row_ids, row_id_kind, columns, name="input", n_rows=None):
        self.row_id, self._row_ids, self.row_id_kind = row_id, row_ids, row_id_kind
        self.columns = list(columns)
        self.name = name
        self.n_rows = len(row_ids) if n_rows is None else int(n_rows)
        self.by_name = {c.name: c for c in self.columns}
        self.row_offset = 0      # first global row of this shard
        self.n_rows_global = self.n_rows

    @property
    def row_ids(self):
        """Host array of the row ids (a device-resident ingest only materialises it when asked)."""
        if callable(self._row_ids):
            self._row_ids = self._row_ids()
        return self._row_ids

    @row_ids.setter
    def row_ids(self, v):
        self._row_ids = v

    @property
    def names(self):
        return [c.name for c in self.columns]

    @property
    def continuous_attrs(self):
        return [c.name for c in self.columns if c.continuous]

    # ---- constructors --------------------------------------------------------------------------
    @classmethod
    def from_pandas(cls, df, row_id, name="input"):
        """checkInputTable (RepairApi.scala:34-67): type gate, >= 3 columns, unique row id."""
        import pandas as pd
        if row_id not in df.columns:
            raise AnalysisException("Column '{}' does not exist in table '{}'".format(row_id, name))
        kinds, bad = {}, []
        for c in df.columns:
            k = df[c].dtype.kind
            if k == "b":
                bad.append("boolean")
            elif k in "iu":
                kinds[c] = "int"
            elif k == "f":
                kinds[c] = "float"
            elif k in "OUS" or str(df[c].dtype) in ("string", "str", "category"):
                kinds[c] = "str"
            elif k == "M":
                bad.append("timestamp")
            else:
                bad.append(str(df[c].dtype))
        if bad:
            raise AnalysisException("Supported types are {}, but unsupported ones found: {}".format(
                _SUPPORTED_MSG, ",".join(bad)))
        # object columns holding only numbers (e.g. nullable ints collected from Spark) are numeric
        for c, k in list(kinds.items()):
            if k == "str" and df[c].dtype == object:
                non_null = [v for v in df[c].tolist() if v is not None and not (isinstance(v, float) and v != v)]
                if non_null and all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in non_null):
                    kinds[c] = "int"
                elif non_null and all(isinstance(v, (int, float, np.integer, np.floating)) and
                                      not isinstance(v, bool) for v in non_null):
                    kinds[c] = "float"
        if not len(df.columns) >= 3:
            raise AnalysisException("A least three columns (`{}` columns + two more ones) in table '{}'".format(
                row_id, name))
        n_distinct = int(df[row_id].nunique(dropna=False))
        if n_distinct != len(df):
            raise AnalysisException(
                "Uniqueness does not hold in column '{}' of table '{}' (# of distinct '{}': {}, # of rows: {})".format(
                    row_id, name, row_id, n_distinct, len(df)))
        cols = []
        for c in df.columns:
            if c == row_id:
                continue
            if kinds[c] == "str":
                cols.append(_encode_strings(c, df[c]))
            else:
                arr = pd.to_numeric(df[c], errors="coerce").to_numpy(dtype=np.float64, na_value=np.nan)
                cols.append(_encode_numeric(c, kinds[c], arr, _numpy_spark_type(df[c].dtype, kinds[c])))
        return cls(row_id, df[row_id].to_numpy(), kinds[row_id], cols, name)

    @classmethod
    def from_arrow(cls, tbl, row_id, name="input"):
        """Same gate and encoding as from_pandas for a ``pyarrow.Table`` (what ``spark_df.toArrow()`` or
        ``pyarrow.parquet.read_table(path, read_dictionary=[...])`` return), without a Python object
        per cell: strings are dictionary-encoded by Arrow's C++ kernels -- columns that already arrive
        dictionary-encoded (Parquet dictionary pages) are NOT decoded first -- and only the
        dictionaries (one entry per distinct value) are sorted and turned into Python strings."""
        import pyarrow as pa
        import pyarrow.compute as pc
        kinds = _arrow_gate(tbl, row_id, name)
        n_distinct = int(pc.count_distinct(tbl[row_id], mode="all").as_py())
        if n_distinct != tbl.num_rows:
            raise AnalysisException(
                "Uniqueness does not hold in column '{}' of table '{}' (# of distinct '{}': {}, # of rows: {})".format(
                    row_id, name, row_id, n_distinct, tbl.num_rows))

        def plain(col):
            col = col.unify_dictionaries() if pa.types.is_dictionary(col.type) else col
            return col.combine_chunks() if col.num_chunks != 1 else col.chunk(0)

        cols = []
        for f in tbl.schema:
            if f.name == row_id:
                continue
            arr = plain(tbl[f.name])
            if kinds[f.name] != "str":
                if pa.types.is_dictionary(arr.type):
                    arr = arr.dictionary_decode()
                vals = pc.cast(arr, pa.float64()).to_numpy(zero_copy_only=False)
                cols.append(_encode_numeric(f.name, kinds[f.name], np.asarray(vals, dtype=np.float64),
                                            _arrow_spark_type(f.type.value_type if pa.types.is_dictionary(f.type)
                                                              else f.type)))
                continue
            cols.append(_encode_arrow_strings(f.name, arr))
        ids = plain(tbl[row_id])
        if pa.types.is_dictionary(ids.type):
            ids = ids.dictionary_decode()
        return cls(row_id, np.asarray(ids.to_numpy(zero_copy_only=False)), kinds[row_id], cols, name)

    @classmethod
    def from_arrow_device(cls, tbl, row_id, ctx, device, name="input", threads=0, timings=None):
        """Device-side ingest of an all-discrete ``pyarrow.Table``: the raw Arrow buffers (dictionary
        indices as int8 / int16 / int32, validity bits, int64 row ids) cross PCIe as they are
        (``dr_h2d_copy``: pageable memory through a pinned chunk ring, several threads), the device finds
        the dictionary entries that occur (``dr_index_presence``), the host sorts the dictionaries (one
        entry per distinct value) and the device rewrites the indices as int32 codes of the sorted
        dictionaries (``dr_index_remap``).  Row-id uniqueness is checked on the device too.  No per-row
        work on the host, no host copy of the codes (``Column.codes`` fetches them on demand).
        -> (EncodedTable, DeviceTable), or None when the table needs the host path of ``from_arrow``
        (numeric attributes, row ids that are not NULL-free integers, an empty table)."""
        import time
        import pyarrow as pa
        import pyarrow.compute as pc
        import torch
        kinds = _arrow_gate(tbl, row_id, name)
        attrs = [f.name for f in tbl.schema if f.name != row_id]
        n = tbl.num_rows
        id_type = tbl.schema.field(row_id).type
        if n == 0 or any(kinds[a] != "str" for a in attrs) or not pa.types.is_integer(id_type) or \
                tbl[row_id].null_count != 0:
            return None
        t0 = time.perf_counter()
        # ---- row ids: to the device, uniqueness there ------------------------------------------------
        ids_col = tbl[row_id] if id_type == pa.int64() else pc.cast(tbl[row_id], pa.int64())
        ids_dev = torch.empty(n, dtype=torch.int64, device=device)
        src, dst, size, off = [], [], [], 0
        for ch in ids_col.chunks:
            if len(ch):
                src.append(ch.buffers()[1].address + ch.offset * 8)
                dst.append(ids_dev.data_ptr() + off * 8)
                size.append(len(ch) * 8)
                off += len(ch)
        ctx.h2d_copy(src, dst, size, threads)
        if not ctx.ids_unique(ids_dev, n):
            n_distinct = int(pc.count_distinct(tbl[row_id], mode="all").as_py())
            raise AnalysisException(
                "Uniqueness does not hold in column '{}' of table '{}' (# of distinct '{}': {}, # of rows: {})".format(
                    row_id, name, row_id, n_distinct, n))
        t_ids = time.perf_counter() - t0
        # ---- attribute columns: what has to travel ---------------------------------------------------
        plan = []   # per attribute: (entries, width, [(idx address, validity address or 0, bit offset, rows)])
        for a in attrs:
            col = tbl[a]
            if not pa.types.is_dictionary(col.type):
                col = pc.dictionary_encode(col)          # plain strings: Arrow's C++ hash kernel, on the host
            if col.num_chunks > 1:
                col = col.unify_dictionaries()
            it = col.type.index_type
            if pa.types.is_unsigned_integer(it) or it.bit_width > 32:
                col = col.cast(pa.dictionary(pa.int32(), col.type.value_type))
                it = pa.int32()
            width = it.bit_width // 8
            chunks = [ch for ch in col.chunks if len(ch)]
            entries = chunks[0].dictionary.to_pylist()
            parts = []
            for ch in chunks:
                bufs = ch.indices.buffers()
                vbuf = ch.buffers()[0] if ch.null_count else None
                parts.append((ch, bufs[1].address + ch.offset * width,
                              (vbuf.address + ch.offset // 8) if vbuf is not None else 0, ch.offset % 8, len(ch)))
            plan.append((entries, width, parts))
        table_cols = [None] * len(attrs)
        n_pad = (n + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN or ROW_ALIGN
        codes = torch.empty((len(attrs), n_pad), dtype=torch.int32, device=device)
        if n_pad > n:
            codes[:, n:].fill_(-1)
        al = lambda b: (b + 255) // 256 * 256
        # Columns travel in groups: while the worker threads copy group g + 1, the device finds the dictionary
        # entries of group g that occur (side stream), and group g's indices are re-encoded as soon as its
        # dictionaries are sorted -- only the last group's encode is not hidden behind a copy.
        budget = 4 << 30   # raw bytes of one group on the device
        side = torch.cuda.Stream(device=device)
        t_copy = t_remap = 0.0
        keep_alive = []
        phases = {"wait_presence_s": 0.0, "sort_dictionaries_s": 0.0, "lut_upload_s": 0.0, "final_sync_s": 0.0}

        def launch_presence(g0, g1, where):
            uoff = [0]
            for i in range(g0, g1):
                uoff.append(uoff[-1] + (len(plan[i][0]) + 31) // 32)
            with torch.cuda.stream(side):
                used = torch.zeros(max(uoff[-1], 1), dtype=torch.int32, device=device)
                for i in range(g0, g1):
                    entries, width, parts = plan[i]
                    if not entries:
                        continue
                    for j, (_, _, _, bo, r) in enumerate(parts):
                        d_idx, d_val = where[(i, j)]
                        ctx.index_presence(d_idx, width, d_val, bo, r, len(entries), used[uoff[i - g0]:])
                used_h = torch.empty(used.shape, dtype=torch.int32, pin_memory=True)
                used_h.copy_(used, non_blocking=True)
                done = torch.cuda.Event()
                done.record(side)
            return uoff, used, used_h, done

        def finish(g0, g1, where, pres):
            """Sorted dictionaries of the group (host, one entry per distinct value) -> LUTs -> re-encode."""
            uoff, used, used_h, done = pres
            t_w = time.perf_counter()
            done.synchronize()
            phases["wait_presence_s"] += time.perf_counter() - t_w
            t_w = time.perf_counter()
            bits_all = used_h.numpy().view(np.uint32)
            luts, loff = [], [0]
            for i in range(g0, g1):
                entries = plan[i][0]
                bits = np.unpackbits(bits_all[uoff[i - g0]:uoff[i - g0 + 1]].view(np.uint8),
                                     bitorder="little")[:len(entries)]
                dictionary, lut = _sorted_dictionary(entries, bits.astype(bool))
                luts.append(lut)
                loff.append(loff[-1] + len(lut))
                table_cols[i] = Column(attrs[i], "str", dictionary, None, None, "string")
            phases["sort_dictionaries_s"] += time.perf_counter() - t_w
            t_w = time.perf_counter()
            with torch.cuda.stream(side):
                d_lut = torch.from_numpy(np.concatenate(luts + [np.zeros(1, dtype=np.int32)])).to(device)
                phases["lut_upload_s"] += time.perf_counter() - t_w
                for i in range(g0, g1):
                    entries, width, parts = plan[i]
                    row = 0
                    for j, (_, _, _, bo, r) in enumerate(parts):
                        d_idx, d_val = where[(i, j)]
                        ctx.index_remap(d_idx, width, d_val, bo, r, d_lut.data_ptr() + 4 * loff[i - g0], len(entries),
                                        codes[i].data_ptr() + 4 * row)
                        row += r
            keep_alive.append((d_lut, used, used_h))

        side.wait_stream(torch.cuda.current_stream())   # (the padding fill of `codes`)
        pending = None
        g0 = 0
        while g0 < len(attrs):
            g1, total = g0, 0
            while g1 < len(attrs) and g1 - g0 < INGEST_GROUP_COLS:
                need = sum(al(r * plan[g1][1]) + (al((r + bo + 7) // 8) if va else 0) for _, _, va, bo, r in plan[g1][2])
                if g1 > g0 and total + need > budget:
                    break
                total += need
                g1 += 1
            stage = torch.empty(max(total, 1), dtype=torch.uint8, device=device)
            keep_alive.append(stage)
            base = stage.data_ptr()
            src, dst, size, where, pos = [], [], [], {}, 0
            for i in range(g0, g1):
                _, width, parts = plan[i]
                for j, (_, ia, va, bo, r) in enumerate(parts):
                    src.append(ia); dst.append(base + pos); size.append(r * width)
                    d_idx = base + pos
                    pos += al(r * width)
                    d_val = 0
                    if va:
                        nb = (r + bo + 7) // 8
                        src.append(va); dst.append(base + pos); size.append(nb)
                        d_val = base + pos
                        pos += al(nb)
                    where[(i, j)] = (d_idx, d_val)
            t1 = time.perf_counter()
            ctx.h2d_copy(src, dst, size, threads)        # blocks; the previous group's kernels run meanwhile
            t_copy += time.perf_counter() - t1
            t1 = time.perf_counter()
            # (the previous group first: its LUT upload is a synchronous copy on the side stream and would
            # otherwise wait for this group's presence kernels, holding back the next group's copy)
            if pending is not None:
                finish(*pending)
            pres = launch_presence(g0, g1, where)
            pending = (g0, g1, where, pres)
            t_remap += time.perf_counter() - t1
            g0 = g1
        t1 = time.perf_counter()
        if pending is not None:
            finish(*pending)
        t_w = time.perf_counter()
        torch.cuda.current_stream().wait_stream(side)
        side.synchronize()
        phases["final_sync_s"] += time.perf_counter() - t_w
        keep_alive.clear()
        t_remap += time.perf_counter() - t1

        def ids_host():
            return np.asarray(ids_col.to_numpy(zero_copy_only=False))
        t = cls(row_id, ids_host, kinds[row_id], table_cols, name, n_rows=n)
        dt = DeviceTable(t, device, codes=codes)
        dt.ids = ids_dev
        for i, c in enumerate(table_cols):
            # the column tensor, not `dt`: dt.table -> t -> closure -> dt would be a reference cycle that keeps
            # the whole device table alive after the run until the cyclic garbage collector happens to run
            c._codes = (lambda col=codes[i]: col[:n].cpu().numpy())
        if timings is not None:
            timings.update({"ingest_copy_s": t_copy, "ingest_encode_s": t_remap,
                            "ingest_total_s": time.perf_counter() - t0, "ingest_ids_s": t_ids,
                            "ingest_encode_phases": dict(phases)})
        return t, dt

    @classmethod
    def from_codes(cls, row_id, names, codes, dict_sizes, name="input", row_ids=None, dictionaries=None):
        """Pre-encoded discrete table (already label-encoded upstream, e.g. Arrow dictionary pages
        or the synthetic generator): ``codes[k]`` int32, -1 = NULL; value c of column k prints as
        ``dictionaries[k][c]`` (default ``"v%03d" % c``)."""
        n = len(codes[0]) if len(codes) else 0
        cols = []
        for i, nm in enumerate(names):
            d = dictionaries[i] if dictionaries is not None else \
                np.array(["v%03d" % c for c in range(int(dict_sizes[i]))], dtype=object)
            cols.append(Column(nm, "str", d, np.ascontiguousarray(codes[i], dtype=np.int32), None))
        if row_ids is None:
            row_ids = np.arange(n, dtype=np.int64)
        if len(names) + 1 < 3:
            raise AnalysisException("A least three columns (`{}` columns + two more ones) in table '{}'".format(
                row_id, name))
        return cls(row_id, row_ids, "int", cols, name)

    def row_id_strings(self, positions):
        ids = self.row_ids[np.asarray(positions, dtype=np.int64)]
        return ids

    def unify(self, dist, device_table=None, ctx=None):
        """Row-sharded input (every rank collected its own rows): makes the dictionaries GLOBAL -- the
        sorted union of the shards' dictionaries, so that a code means the same value on every GPU and
        the count tensors of the shards add up -- and records the shard's place in the global table.
        Only dictionaries (one entry per distinct value) and row counts cross the wire.  With a
        `device_table` (device-side Arrow ingest) the resident codes are re-labelled in place on the
        device (dr_index_remap) and no host copy of them is made."""
        import torch.distributed as td
        local = [(c.name, c.kind, list(c.dictionary) if c.kind == "str" else np.asarray(c.dictionary, dtype=np.float64))
                 for c in self.columns]
        gathered = [None] * dist.world
        td.all_gather_object(gathered, (self.n_rows, local), group=dist.group)
        names = [nm for nm, _, _ in local]
        for n_r, cols in gathered:
            if [nm for nm, _, _ in cols] != names:
                raise AnalysisException("the shards of table '{}' do not have the same columns".format(self.name))
        counts = [n_r for n_r, _ in gathered]
        cols = []
        for i, c in enumerate(self.columns):
            kinds = {g[1][i][1] for g in gathered}
            kind = c.kind if len(kinds) == 1 else ("float" if kinds <= {"int", "float"} else "str")
            if kind == "str":
                merged = np.array(sorted(set(str(v) for g in gathered for v in g[1][i][2])), dtype=object)
                mine = np.array([str(v) for v in c.dictionary], dtype=object)
                lut = np.searchsorted(merged.astype(str), mine.astype(str)).astype(np.int32) if len(mine) else \
                    np.zeros(0, dtype=np.int32)
                values = None
            else:
                merged = np.unique(np.concatenate([np.asarray(g[1][i][2], dtype=np.float64) for g in gathered]))
                lut = np.searchsorted(merged, np.asarray(c.dictionary, dtype=np.float64)).astype(np.int32)
                values = c.values
            if device_table is not None:
                import torch
                col = device_table.codes[device_table.col_index[c.name]]
                if len(lut) and not np.array_equal(lut, np.arange(len(lut))):
                    d_lut = torch.from_numpy(lut).to(col.device)
                    ctx.index_remap(col.data_ptr(), 4, 0, 0, self.n_rows, d_lut.data_ptr(), len(lut), col.data_ptr())
                    torch.cuda.current_stream().synchronize()   # d_lut is released on return
                codes = (lambda col=col, n=self.n_rows: col[:n].cpu().numpy())
            else:
                codes = np.where(c.codes >= 0, np.r_[lut, np.int32(-1)][c.codes], -1).astype(np.int32) if len(lut) else \
                    np.full(len(c.codes), -1, dtype=np.int32)
            cols.append(Column(c.name, kind, merged, codes, values,
                               c.spark_type if len(kinds) == 1 else None))
        t = EncodedTable(self.row_id, self._row_ids, self.row_id_kind, cols, self.name, n_rows=self.n_rows)
        t.row_offset = int(sum(counts[:dist.rank]))
        t.n_rows_global = int(sum(counts))
        if device_table is not None:
            device_table.table = t
        return t

    def shard(self, rank, world):
        """Contiguous row shard [lo, hi) for rank `rank` of `world` (global dictionaries kept)."""
        n = self.n_rows
        lo, hi = (n * rank) // world, (n * (rank + 1)) // world
        cols = [Column(c.name, c.kind, c.dictionary, c.codes[lo:hi], None if c.values is None else c.values[lo:hi],
                       c.spark_type) for c in self.columns]
        t = EncodedTable(self.row_id, self.row_ids[lo:hi], self.row_id_kind, cols, self.name)
        t.row_offset, t.n_rows_global = lo, n
        return t


class DeviceTable:
    """The encoded table resident in HBM: ``codes`` int32 [K][n_pad] (one contiguous column per
    attribute) and ``values`` float64 [Kc][n_pad] for the continuous attributes."""

    def __init__(self, table, device, codes=None, values=None, ctx=None):
        import torch
        self.table = table
        self.device = device
        self.n_rows = table.n_rows
        self.n_pad = (self.n_rows + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN or ROW_ALIGN
        K = len(table.columns)
        self.cont_index = {c.name: i for i, c in enumerate([c for c in table.columns if c.continuous])}
        if codes is None:
            codes = torch.empty((K, self.n_pad), dtype=torch.int32, device=device)
            staging = torch.empty((self.n_pad,), dtype=torch.int32).pin_memory()
            narrow = narrow_dev = None
            for i, c in enumerate(table.columns):
                if c.dict_size <= 254 and ctx is not None:
                    # small dictionaries cross PCIe as one byte per cell and are widened on the device
                    if narrow is None:
                        narrow = torch.empty((self.n_pad,), dtype=torch.uint8).pin_memory()
                        narrow_dev = torch.empty((self.n_pad,), dtype=torch.uint8, device=device)
                    narrow[:self.n_rows].copy_(torch.from_numpy(np.ascontiguousarray(c.codes).astype(np.uint8)))
                    narrow[self.n_rows:].fill_(255)
                    narrow_dev.copy_(narrow, non_blocking=True)
                    ctx.widen_u8(narrow_dev, self.n_pad, codes[i])
                else:
                    staging[:self.n_rows].copy_(torch.from_numpy(np.ascontiguousarray(c.codes)))
                    staging[self.n_rows:].fill_(-1)
                    codes[i].copy_(staging, non_blocking=True)
                torch.cuda.current_stream().synchronize()
        self.codes = codes
        if values is None and self.cont_index:
            values = torch.empty((len(self.cont_index), self.n_pad), dtype=torch.float64, device=device)
            staging = torch.empty((self.n_pad,), dtype=torch.float64).pin_memory()
            for c in table.columns:
                if c.continuous:
                    staging[:self.n_rows].copy_(torch.from_numpy(np.array(c.values, dtype=np.float64)))  # (own, writable copy)
                    staging[self.n_rows:].fill_(float("nan"))
                    values[self.cont_index[c.name]].copy_(staging, non_blocking=True)
                    torch.cuda.current_stream().synchronize()
        self.values = values
        self.col_index = {c.name: i for i, c in enumerate(table.columns)}
        self.ids = None   # device int64 row ids (device-side Arrow ingest), else None

    def col(self, name):
        return self.codes[self.col_index[name]]

    def val(self, name):
        return self.values[self.cont_index[name]]


class ByteStager:
    """Ingest of successive batches of an all-small-dictionary table (every dictionary <= 254 entries,
    one byte per cell in pinned host memory, 255 = NULL) into ONE resident DeviceTable: the host->device
    copy of batch i + 1 runs on its own stream into the other of two device staging buffers while
    batch i is being processed, so PCIe time leaves the critical path; what stays on it is the
    widening pass (dr_widen_u8: 1 B read + 4 B written per cell)."""

    def __init__(self, device_table, ctx):
        import torch
        self.torch, self.dt, self.ctx = torch, device_table, ctx
        shape = tuple(device_table.codes.shape)
        self.stage = [torch.empty(shape, dtype=torch.uint8, device=device_table.device) for _ in range(2)]
        self.copied = [torch.cuda.Event(), torch.cuda.Event()]     # H2D of the buffer finished
        self.consumed = [torch.cuda.Event(), torch.cuda.Event()]   # widening pass read the buffer
        self.stream = torch.cuda.Stream(device=device_table.device)
        self.pending = [False, False]
        self.n = 0                                                  # batches handed to the table so far

    def prefetch(self, host_bytes):
        """Start copying the NEXT batch (pinned uint8 [K][n_pad]) to the device."""
        j = (self.n + (1 if self.pending[self.n % 2] else 0)) % 2
        assert not self.pending[j], "both staging buffers are in flight"
        self.stream.wait_event(self.consumed[j])
        with self.torch.cuda.stream(self.stream):
            self.stage[j].copy_(host_bytes, non_blocking=True)
            self.copied[j].record(self.stream)
        self.pending[j] = True

    def next_batch(self, host_bytes=None):
        """Make the oldest prefetched batch (or `host_bytes`, copied now) the table's content."""
        j = self.n % 2
        if not self.pending[j]:
            assert host_bytes is not None, "nothing prefetched"
            self.prefetch(host_bytes)
        main = self.torch.cuda.current_stream()
        main.wait_event(self.copied[j])
        self.ctx.widen_u8(self.stage[j], self.stage[j].numel(), self.dt.codes)
        self.consumed[j].record(main)
        self.pending[j] = False
        self.n += 1


def cells_to_arrow(table, cells):
    """Egress without a Python string per cell: the (row id, attribute, current_value, repaired) frame of
    encoded repair output ``[(attr, row positions, current codes, repaired codes)]`` as a pyarrow.Table
    whose string columns are dictionary arrays over the column dictionaries (one chunk per attribute)."""
    import pyarrow as pa
    names = [a for a, _, _, _ in cells]
    ids, attr_idx, cur, rep = [], [], [], []
    for i, (a, rows, c, r) in enumerate(cells):
        col = table.by_name[a]
        if col.kind != "str":
            raise NotImplementedError("cells_to_arrow takes discrete attributes (dictionary codes)")
        strs = pa.array(col.strings(), type=pa.string())
        ids.append(pa.array(table.row_ids[np.asarray(rows, dtype=np.int64)]))
        attr_idx.append(np.full(len(rows), i, dtype=np.int32))
        for codes, out in ((c, cur), (r, rep)):
            codes = np.asarray(codes, dtype=np.int32)
            out.append(pa.DictionaryArray.from_arrays(pa.array(codes, mask=codes < 0), strs))
    if not cells:
        empty = pa.array([], type=pa.string())
        return pa.table({table.row_id: pa.array(table.row_ids[:0]), "attribute": empty, "current_value": empty,
                         "repaired": empty})
    attribute = pa.DictionaryArray.from_arrays(pa.array(np.concatenate(attr_idx)), pa.array(names, type=pa.string()))
    return pa.table({table.row_id: pa.chunked_array(ids), "attribute": attribute,
                     "current_value": pa.chunked_array(cur), "repaired": pa.chunked_array(rep)})

