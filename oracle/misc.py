"""NumPy / pandas restatement of the delphi.misc utilities (RepairMiscApi.scala:41-347), written from the
Spark SQL of the reference and independently of ``repair.misc`` / ``repair.cluster``: every answer is
computed from the frame's cells, and splitInputTable's q-gram bags are built per row as explicit sparse
vectors, with ||x - mu||^2 taken from those vectors."""
import math
from decimal import Decimal

import numpy as np
import pandas as pd
import scipy.sparse as sp

VOCAB_CAP = 1 << 18


def _is_null(v):
    return v is None or v is pd.NA or (isinstance(v, float) and v != v)


def _java_double(v):
    """Java's Double.toString."""
    if v == 0.0:
        return "-0.0" if math.copysign(1.0, v) < 0 else "0.0"
    if math.isinf(v):
        return "Infinity" if v > 0 else "-Infinity"
    sign, digits, exp = Decimal(repr(abs(v))).normalize().as_tuple()
    ds = "".join(map(str, digits))
    lead = len(ds) + exp - 1
    mag = abs(v)
    s = "-" if v < 0 else ""
    if 1e-3 <= mag < 1e7:
        if lead < 0:
            return s + "0." + "0" * (-lead - 1) + ds
        whole = ds[:lead + 1].ljust(lead + 1, "0")
        return s + whole + "." + (ds[lead + 1:] or "0")
    return "{}{}.{}E{}".format(s, ds[0], ds[1:] or "0", lead)


def _numeric_kind(s):
    k = s.dtype.kind
    return "int" if k in "iu" else "float" if k == "f" else None


def cast_string(s, as_double=False):
    """CAST(column AS STRING) -> list (None for NULL); as_double: the column is first cast to DOUBLE."""
    kind = _numeric_kind(s)
    if as_double and kind == "int":
        kind = "float"
    out = []
    for v in s.tolist():
        if _is_null(v):
            out.append(None)
        elif kind == "int":
            out.append(str(int(v)))
        elif kind == "float":
            out.append(_java_double(float(v)))
        else:
            out.append(str(v))
    return out


def describe(df, num_bins=8):
    rows = []
    for c in df.columns:
        s = df[c]
        kind = _numeric_kind(s)
        present = [v for v in s.tolist() if not _is_null(v)]
        mn = mx = hist = None
        if kind:
            size = s.dtype.itemsize
            avg = mxl = size
            if present:
                vals = sorted(float(v) for v in present)
                f = (lambda v: str(int(v))) if kind == "int" else _java_double
                mn, mx = f(vals[0]), f(vals[-1])
                n = len(vals)
                pct = [vals[max(1, math.ceil(i * n / num_bins)) - 1] for i in range(num_bins + 1)]
                gaps = np.diff(np.array(pct))
                with np.errstate(invalid="ignore", divide="ignore"):
                    hist = (gaps / gaps.sum()).tolist()
        else:
            strs = [str(v) for v in present]
            if strs:
                avg = math.ceil(sum(len(x) for x in strs) / len(strs))
                mxl = max(len(x) for x in strs)
            else:
                avg = mxl = 20
        rows.append((str(c), len(set(present)), mn, mx, len(s) - len(present), avg, mxl, hist))
    names = ["attrName", "distinctCnt", "min", "max", "nullCnt", "avgLen", "maxLen", "hist"]
    return pd.DataFrame({c: pd.Series([r[i] for r in rows], dtype=object if c in ("attrName", "min", "max", "hist")
                                       else np.int64) for i, c in enumerate(names)})


def to_histogram(df, targets):
    want = {t.strip() for t in targets.split(",") if t.strip()}
    rows = []
    for c in df.columns:
        if c in want and _numeric_kind(df[c]) is None:
            vc = {}
            for v in df[c].tolist():
                if not _is_null(v):
                    vc[str(v)] = vc.get(str(v), 0) + 1
            rows.append((c, [{"value": v, "cnt": vc[v]} for v in sorted(vc)]))
    return pd.DataFrame(rows, columns=["attribute", "histogram"])


def to_error_map(df, row_id, cells):
    errs = {(str(r), str(a)) for r, a in zip(cells[row_id].tolist(), cells["attribute"].tolist())}
    attrs = [c for c in df.columns if c != row_id]
    maps = ["".join("*" if (str(r), a) in errs else "-" for a in attrs) for r in df[row_id].tolist()]
    return pd.DataFrame({row_id: df[row_id].to_numpy(), "error_map": maps})


def flatten(df, row_id):
    attrs = [c for c in df.columns if c != row_id]
    K, n = len(attrs), len(df)
    vals = np.empty((n, K), dtype=object)
    for j, a in enumerate(attrs):
        vals[:, j] = cast_string(df[a])
    return pd.DataFrame({row_id: np.repeat(df[row_id].to_numpy(), K),
                         "attribute": np.tile(np.array(attrs, dtype=object), n), "value": vals.reshape(-1)})


def mix(seed, col, rows):
    """splitmix64 of repair/synth.py: top 53 bits."""
    from repair.synth import _mix_np
    return _mix_np(seed, col, np.asarray(rows, dtype=np.int64))


def inject_null_keep(seed, col, n, ratio):
    """rand() > ratio per row of schema column `col` (before the cell's own NULL)."""
    return mix(seed, col, np.arange(n)).astype(np.float64) * 2.0 ** -53 > ratio


def inject_null(df, targets, ratio, seed):
    out = df.copy()
    for ci, c in enumerate(df.columns):
        if c in targets:
            keep = inject_null_keep(seed, ci, len(df), ratio) & ~pd.isna(df[c]).to_numpy()
            out[c] = [v if k else None for v, k in zip(df[c].tolist(), keep.tolist())]
    return out


# ---- splitInputTable -----------------------------------------------------------------------------------
def qgrams(s, q):
    return [s[i:i + q] for i in range(len(s) - q + 1)] if len(s) > q else [s]


def bags(df, targets, q):
    """Per-row q-gram bags -> (sparse rows x terms, terms) in the canonical term order (total count
    descending, then the term), capped at 2^18 terms."""
    per_row = [dict() for _ in range(len(df))]
    # array(targets) has one element type: all-numeric targets with a floating one are all DOUBLE
    kinds = [_numeric_kind(df[t]) for t in targets]
    as_double = None not in kinds and "float" in kinds
    for t in targets:
        for r, s in enumerate(cast_string(df[t], as_double)):
            if s is None:
                continue
            bag = per_row[r]
            for g in qgrams(s, q):
                bag[g] = bag.get(g, 0) + 1
    total = {}
    for bag in per_row:
        for g, m in bag.items():
            total[g] = total.get(g, 0) + m
    terms = sorted(total, key=lambda g: (-total[g], g))[:VOCAB_CAP]
    tid = {g: i for i, g in enumerate(terms)}
    rows, cols, vals = [], [], []
    for r, bag in enumerate(per_row):
        for g, m in bag.items():
            if g in tid:
                rows.append(r)
                cols.append(tid[g])
                vals.append(m)
    x = sp.csr_matrix((np.array(vals, dtype=np.float64), (np.array(rows, dtype=np.int64),
                                                          np.array(cols, dtype=np.int64))),
                      shape=(len(df), len(terms)))
    return x, terms


def sq_dist(x, centres):
    """||x_r - mu_j||^2 for every row and centre."""
    x_sq = np.asarray(x.multiply(x).sum(axis=1)).ravel()
    mu_sq = (centres ** 2).sum(axis=1)
    return np.maximum(x_sq[:, None] - 2.0 * np.asarray(x @ centres.T) + mu_sq[None, :], 0.0)


def _means(x, labels, ids, old):
    new = old.copy()
    for j in ids:
        m = labels == j
        if m.any():
            new[j] = np.asarray(x[m].sum(axis=0)).ravel() / m.sum()
    return new


def kmeans(x, init, max_iter=20, tol=1e-4):
    """Lloyd's algorithm from `init` -> (labels, iterations, centres); the labels are the assignment to the
    final centres; stop when no centre moved more than tol."""
    centres = np.array(init, dtype=np.float64)
    it = 0
    while it < max_iter:
        labels = np.argmin(sq_dist(x, centres), axis=1)
        new = _means(x, labels, range(len(centres)), centres)
        moved = ((new - centres) ** 2).sum(axis=1)
        centres = new
        it += 1
        if np.all(moved <= tol * tol):
            break
    return np.argmin(sq_dist(x, centres), axis=1), it, centres


def bisecting_kmeans(x, k, max_iter=20, seed=0):
    """Spark's BisectingKMeans (minDivisibleClusterSize 1): levels of simultaneous splits of the clusters made
    on the previous level, the largest first when fewer are needed; children of node i are 2i and 2i + 1,
    started at mu -/+ 1e-4 ||mu|| u with u = default_rng([seed, i]).random(terms); a split counts only when
    both children get rows.  -> leaf index per row, leaves numbered depth first."""
    n, d = x.shape
    node = np.ones(n, dtype=np.int64)
    centre = {1: np.asarray(x.sum(axis=0)).ravel() / max(n, 1)}
    size = {1: n}
    children = {}
    active, needed = [1], k - 1
    while active and needed > 0:
        div = [i for i in active if size[i] >= 2]
        if len(div) > needed:
            div = sorted(div, key=lambda i: (-size[i], i))[:needed]
        if not div:
            break
        cen = {}
        for i in div:
            level = 1e-4 * np.sqrt(centre[i] @ centre[i])
            u = np.random.default_rng([seed, i]).random(d)
            cen[2 * i], cen[2 * i + 1] = centre[i] - level * u, centre[i] + level * u
        rows = {i: np.nonzero(node == i)[0] for i in div}

        def assign():
            lab = {}
            for i in div:
                dd = sq_dist(x[rows[i]], np.array([cen[2 * i], cen[2 * i + 1]]))
                lab[i] = np.where(dd[:, 1] < dd[:, 0], 2 * i + 1, 2 * i)
            return lab

        for _ in range(max_iter):
            lab = assign()
            for i in div:
                for ch in (2 * i, 2 * i + 1):
                    m = lab[i] == ch
                    if m.any():
                        cen[ch] = np.asarray(x[rows[i][m]].sum(axis=0)).ravel() / m.sum()
        lab = assign()
        active = []
        for i in div:
            node[rows[i]] = lab[i]
            kids = [ch for ch in (2 * i, 2 * i + 1) if (lab[i] == ch).any()]
            children[i] = kids
            for ch in kids:
                size[ch] = int((lab[i] == ch).sum())
                centre[ch] = cen[ch]
            if len(kids) == 2:
                active += kids
                needed -= 1
    leaf, order = {}, [1]
    while order:
        i = order.pop()
        if children.get(i):
            order += children[i][::-1]
        else:
            leaf[i] = len(leaf)
    return np.array([leaf[i] for i in node.tolist()], dtype=np.int32)


def assign_from_p(codes, dom, p_off, P, mu_sq, labels=None, split=None):
    """What dr_kmeans_assign computes, restated in NumPy: the dot products summed over the columns in order
    from 0.0, score mu_sq - 2 dot, first minimum; with `split`, only rows whose label L has split[L] >= 0 move
    (to split[L] or split[L] + 1)."""
    n = len(codes[0]) if len(codes) else 0
    slots = [p_off[c] + np.minimum(np.asarray(codes[c], dtype=np.int64) + 1, dom[c]) for c in range(len(codes))]
    if split is None:
        dot = np.zeros((n, P.shape[1]))
        for s in slots:
            dot = dot + P[s]
        return np.argmin(mu_sq[None, :] - 2.0 * dot, axis=1).astype(np.int32)
    labels = np.asarray(labels, dtype=np.int32).copy()
    ok = (labels >= 0) & (labels < len(split))
    s = np.where(ok, np.asarray(split)[np.clip(labels, 0, len(split) - 1)], -1)
    ok &= (s >= 0) & (s + 1 < P.shape[1])
    s = np.where(ok, s, 0)
    a0 = np.zeros(n)
    a1 = np.zeros(n)
    for sl in slots:
        a0 = a0 + P[sl, s]
        a1 = a1 + P[sl, s + 1]
    pick = np.where((mu_sq[s + 1] - 2.0 * a1) < (mu_sq[s] - 2.0 * a0), s + 1, s)
    labels[ok] = pick[ok]
    return labels
