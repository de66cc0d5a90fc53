"""Oracle of LOFOutlierErrorDetector (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Restates ``errors.py:219-245`` with ``LocalOutlierFactor(novelty=False)`` at its defaults over the
column's distinct values with multiplicities (one dimension: a point's k nearest neighbours are a
contiguous run of the sorted order, so all copies of a value share kdist / lrd / lof):

* NULL cells are copies of the median of the non-NULL cells;
* entry i's neighbours: ``cnt[i] - 1`` copies of itself, then whole runs outward, nearest first, an
  equal-distance tie taking the smaller value first; the last run may be partial;
* ``kdist_i`` = distance of the run that completes k;
* ``lrd_i = 1 / (sum_j m_ij * max(d(i,j), kdist_j) / k + 1e-10)``;
* ``lof_i = sum_j m_ij * (lrd_j / lrd_i) / k``;  outlier iff ``lof_i > 1.5``.

Sums run over the window in ascending value order with one rounding per operation (no FMA), the
order ``csrc/lof.cu`` uses, so the GPU must match these arrays bit for bit.
"""
import numpy as np

N_NEIGHBORS = 20          # LocalOutlierFactor's default
CHUNK = 1 << 20           # entries per vectorised step


def effective_k(n_rows):
    return max(1, min(N_NEIGHBORS, n_rows - 1))


def _windows(u, cnt, k, lo_e, hi_e, seg_lo, seg_hi):
    """Windows of entries [lo_e, hi_e) -> (lo, hi, m_lo, m_hi, m_self, kdist), all vectorised.  Entry e only
    sees entries of its own segment [seg_lo[e], seg_hi[e])."""
    D = len(u)
    e = np.arange(lo_e, hi_e, dtype=np.int64)
    s_lo, s_hi = seg_lo[lo_e:hi_e], seg_hi[lo_e:hi_e]
    m_self = np.clip(cnt[e] - 1, 0, k)
    rem = k - m_self
    lo, hi = e.copy(), e.copy()
    m_lo = np.zeros(len(e), dtype=np.int64)
    m_hi = np.zeros(len(e), dtype=np.int64)
    kd = np.zeros(len(e), dtype=np.float64)
    l, r = e - 1, e + 1
    ue = u[e]
    for _ in range(2 * k):
        act = rem > 0
        if not act.any():
            break
        has_l = act & (l >= s_lo) & (l >= e - k)
        has_r = act & (r < s_hi) & (r <= e + k)
        dl = np.where(has_l, ue - u[np.clip(l, 0, D - 1)], 0.0)
        dr = np.where(has_r, u[np.clip(r, 0, D - 1)] - ue, 0.0)
        take_l = has_l & (~has_r | (dl <= dr))
        take_r = has_r & ~take_l
        c = np.where(take_l, cnt[np.clip(l, 0, D - 1)], np.where(take_r, cnt[np.clip(r, 0, D - 1)], 0))
        m = np.minimum(c, rem)
        rem = rem - np.where(take_l | take_r, m, 0)
        kd = np.where(take_l, dl, np.where(take_r, dr, kd))
        lo = np.where(take_l, l, lo)
        m_lo = np.where(take_l, m, m_lo)
        hi = np.where(take_r, r, hi)
        m_hi = np.where(take_r, m, m_hi)
        l = np.where(take_l, l - 1, l)
        r = np.where(take_r, r + 1, r)
        rem = np.where(act & ~(has_l | has_r), 0, rem)   # (cannot happen when every count is >= 1)
    return lo, hi, m_lo, m_hi, m_self, kd


def _window_sum(u, cnt, k, lo_e, hi_e, win, x, pass_):
    """pass_ 1: sum_j m * max(d, x_j) (x = kdist);  pass_ 2: sum_j m * (x_j / x_e) (x = lrd)."""
    D = len(u)
    lo, hi, m_lo, m_hi, m_self, _ = win
    e = np.arange(lo_e, hi_e, dtype=np.int64)
    ue = u[e]
    s = np.zeros(len(e), dtype=np.float64)
    for o in range(-k, k + 1):
        j = e + o
        inc = (j >= lo) & (j <= hi)
        jc = np.clip(j, 0, D - 1)
        m = np.where(o == 0, m_self, np.where(j == lo, m_lo, np.where(j == hi, m_hi, cnt[jc]))).astype(np.float64)
        if pass_ == 1:
            d = ue - u[jc] if o < 0 else (u[jc] - ue if o > 0 else np.zeros(len(e)))
            term = m * np.maximum(d, x[jc])
        else:
            term = m * (x[jc] / x[e])
        s = s + np.where(inc, term, 0.0)
    return s


def lof_entries(u, cnt, k, seg_lo=None, seg_hi=None):
    """u float64[D] strictly ascending, cnt int64[D] >= 1 -> (kdist, lrd, lof, verdict) float64 / bool [D].
    seg_lo / seg_hi (int64[D], optional): u is a concatenation of independent columns and entry e belongs
    to the one spanning [seg_lo[e], seg_hi[e]) (see lof_at)."""
    u = np.ascontiguousarray(u, dtype=np.float64)
    cnt = np.ascontiguousarray(cnt, dtype=np.int64)
    D = len(u)
    if seg_lo is None:
        seg_lo, seg_hi = np.zeros(D, dtype=np.int64), np.full(D, D, dtype=np.int64)
    kdist = np.zeros(D, dtype=np.float64)
    lrd = np.zeros(D, dtype=np.float64)
    lof = np.zeros(D, dtype=np.float64)
    wins = {}
    for a in range(0, D, CHUNK):
        b = min(D, a + CHUNK)
        w = _windows(u, cnt, k, a, b, seg_lo, seg_hi)
        kdist[a:b] = w[5]
        wins[a] = w
    with np.errstate(over="ignore"):
        for a in range(0, D, CHUNK):
            b = min(D, a + CHUNK)
            s = _window_sum(u, cnt, k, a, b, wins[a], kdist, 1)
            lrd[a:b] = 1.0 / (s / float(k) + 1e-10)
        for a in range(0, D, CHUNK):
            b = min(D, a + CHUNK)
            lof[a:b] = _window_sum(u, cnt, k, a, b, wins[a], lrd, 2) / float(k)
    return kdist, lrd, lof, lof > 1.5


def neighbourhoods(D, k, idx):
    """The +-3k neighbourhoods of entries idx of a D-entry column, concatenated: -> (entry indices int64[M],
    seg_lo int64[M], seg_hi int64[M], position of every idx entry in the concatenation)."""
    idx = np.asarray(idx, dtype=np.int64)
    a, b = np.maximum(0, idx - 3 * k), np.minimum(D, idx + 3 * k + 1)
    ln = b - a
    start = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    seg = np.repeat(np.arange(len(idx)), ln)
    flat = a[seg] + (np.arange(int(ln.sum()), dtype=np.int64) - start[seg])
    return flat, start[seg], (start + ln)[seg], start + (idx - a)


def lof_at(u_flat, cnt_flat, seg_lo, seg_hi, k, centres):
    """(kdist, lrd, lof, verdict) of the centre entries of concatenated neighbourhoods (neighbourhoods()):
    lof_i depends on nothing farther than 3k from i, so every centre's values are exact, while a whole
    column of 10^8 entries need not be restated to check a sample of it."""
    kd, lrd, lof, v = lof_entries(u_flat, cnt_flat, k, seg_lo, seg_hi)
    return kd[centres], lrd[centres], lof[centres], v[centres]


def lof_entry(u, cnt, k, i):
    """(kdist, lrd, lof, verdict) of entry i alone, from its +-3k neighbourhood."""
    flat, s_lo, s_hi, centre = neighbourhoods(len(u), k, [i])
    kd, lrd, lof, v = lof_at(np.asarray(u)[flat], np.asarray(cnt)[flat], s_lo, s_hi, k, centre)
    return kd[0], lrd[0], lof[0], bool(v[0])


def weighted_column(vals):
    """float64 column with NaN = NULL -> (u, cnt, k, entry of every row) or None (no cells: fewer than
    two rows, or no non-NULL value).  Raises ValueError on +-inf, as scikit-learn's input check does."""
    vals = np.asarray(vals, dtype=np.float64)
    n = len(vals)
    nul = np.isnan(vals)
    valid = vals[~nul]
    if n < 2 or len(valid) == 0:
        return None
    if np.isinf(valid).any():
        raise ValueError("column contains infinity")
    median = float(np.median(valid))
    filled = np.where(nul, median, vals)
    u, inv, cnt = np.unique(filled, return_inverse=True, return_counts=True)
    return u, cnt.astype(np.int64), effective_k(n), inv


def lof_cells(tbl, row_id, continuous, targets):
    """-> set of (row position, attribute) flagged by LOFOutlierErrorDetector."""
    out = set()
    for attr in [a for a in continuous if a in targets]:
        if attr not in tbl.cols or attr == row_id:
            continue
        got = weighted_column(tbl.cols[attr])
        if got is None:
            continue
        u, cnt, k, inv = got
        verdict = lof_entries(u, cnt, k)[3]
        for r in np.nonzero(verdict[inv])[0]:
            out.add((int(r), attr))
    return out
