"""splitInputTable's clustering (RepairMiscApi.scala:75-153) restated over dictionary codes.

The reference turns each row into the bag of q-grams of its target cells (CountVectorizer) and runs
Spark MLlib's KMeans or BisectingKMeans on those vectors.  Row r's bag is x_r = sum_c B_c[code_c(r)],
where B_c is the (dictionary entry x term) q-gram count matrix of column c, so nothing here is ever
done per row on the host:

* assignment: argmin_j ||x_r - mu_j||^2 = argmin_j (||mu_j||^2 - 2 sum_c P_c[code_c(r), j]) with
  P_c = B_c mu^T, a (dom_c + 1) x k table -- the ``dr_kmeans_assign`` kernel reads K codes per row and
  gathers K rows of P;
* centre update: mu_j = (1 / n_j) sum_c sum_v N_c[j, v] B_c[v], where N_c[j, v] counts the rows with
  label j and code v in column c -- the co-occurrence table of (label column, column c), ``dr_cooc``.

The B_c, P and centre arithmetic run on the host in float64 (one row per dictionary entry, one column
per centre).  Deviations from Spark, all forced by Spark's own random streams or JVM types:

* KMeans starts from k-means++ (D^2 sampling) over a sample of at most 10 000 rows drawn with
  ``numpy.random.default_rng(0)`` instead of Spark's k-means|| initialisation.  This sample is the only
  place row vectors are built.
* BisectingKMeans splits a centre mu into mu -/+ 1e-4 ||mu|| noise with uniform [0, 1) noise from
  ``numpy.random.default_rng([0, node])`` (node: 1 for the root, 2i and 2i + 1 for the children of i)
  instead of a java.util.Random stream.  A leaf is divisible when it holds at least two rows and its
  split leaves both children non-empty; this stands in for Spark's cost > 1e-8 * size test (both
  reject a cluster of identical points).
* Above 2^18 distinct terms the vocabulary keeps the terms with the largest total count over the
  table's cells (Spark ranks by the number of rows that contain a term).
* q-grams are taken over Python code points; Java slices UTF-16 units, so strings with characters
  outside the Basic Multilingual Plane give other q-grams.
"""
import time

import numpy as np
import scipy.sparse as sp

VOCAB_CAP = 1 << 18
MAX_ITER = 20
TOL = 1e-4
SAMPLE_ROWS = 10_000
SEED = 0


def qgrams(s, q):
    """computeQgram (RepairMiscApi.scala:52-71) of one string."""
    if len(s) > q:
        return [s[i:i + q] for i in range(len(s) - q + 1)]
    return [s]


class QgramFeatures:
    """B_c for every target column over one vocabulary, in the canonical term order (total count over the
    table's cells descending, then the term), capped at VOCAB_CAP terms.

    strings[c]: CAST(.. AS STRING) of column c's dictionary entries; hist[c]: int64 counts per slot
    (slot 0 = NULL, slot v + 1 = entry v), as ``dr_scan_hist`` produces them."""

    def __init__(self, strings, hist, q):
        term_id, parts = {}, []
        for strs in strings:
            rows, cols, vals = [], [], []
            for v, s in enumerate(strs):
                bag = {}
                for g in qgrams(s, q):
                    bag[g] = bag.get(g, 0) + 1
                for g, m in bag.items():
                    rows.append(v + 1)
                    cols.append(term_id.setdefault(g, len(term_id)))
                    vals.append(m)
            parts.append((rows, cols, vals, len(strs) + 1))
        n_terms = len(term_id)
        full = [sp.csr_matrix((np.asarray(vals, dtype=np.float64), (np.asarray(rows, dtype=np.int64),
                                                                     np.asarray(cols, dtype=np.int64))),
                              shape=(n1, n_terms)) for rows, cols, vals, n1 in parts]
        total = np.zeros(n_terms, dtype=np.float64)
        for b, h in zip(full, hist):
            total += b.T @ np.asarray(h, dtype=np.float64)
        terms = [None] * n_terms
        for g, t in term_id.items():
            terms[t] = g
        order = sorted(range(n_terms), key=lambda t: (-total[t], terms[t]))[:VOCAB_CAP]
        order = np.asarray(order, dtype=np.int64)
        self.terms = [terms[t] for t in order.tolist()]
        self.B = [b[:, order].tocsr() for b in full]
        self.dom = [b.shape[0] - 1 for b in self.B]
        self.p_off = np.concatenate([[0], np.cumsum([b.shape[0] for b in self.B])[:-1]]).astype(np.int64)
        self.n_terms = len(order)

    def rows(self, codes):
        """Explicit bag vectors (sparse, one row per entry of codes[c]) -- used only for the k-means++ sample."""
        x = None
        for b, cc in zip(self.B, codes):
            part = b[np.asarray(cc, dtype=np.int64) + 1]
            x = part if x is None else x + part
        return x.tocsr()

    def p_table(self, centres):
        """P = [B_c mu^T for every column c] stacked: float64 [sum(dom_c + 1)][k], plus ||mu_j||^2."""
        mu = np.ascontiguousarray(centres, dtype=np.float64)
        P = np.concatenate([np.asarray(b @ mu.T) for b in self.B], axis=0) if self.B else np.zeros((0, len(mu)))
        mu_sq = np.einsum("ij,ij->i", mu, mu)
        return np.ascontiguousarray(P, dtype=np.float64), mu_sq

    def centres_from_counts(self, counts, old):
        """mu_j = (1 / n_j) sum_c N_c[j] B_c; counts[c]: int64 [n_centres][dom_c + 1].  Empty clusters keep
        their centre.  -> (centres, n_j)."""
        n_j = np.asarray(counts[0], dtype=np.int64).sum(axis=1)
        s = np.zeros((len(n_j), self.n_terms), dtype=np.float64)
        for b, n in zip(self.B, counts):
            s += np.asarray((b.T @ np.asarray(n, dtype=np.float64).T).T)
        new = np.array(old, dtype=np.float64, copy=True)
        live = n_j > 0
        new[live] = s[live] / n_j[live, None].astype(np.float64)
        return new, n_j


def kmeanspp(x, k, rng):
    """k-means++ (D^2 sampling) over the rows of sparse x -> dense [k][n_terms]."""
    m = x.shape[0]
    x_sq = np.asarray(x.multiply(x).sum(axis=1)).ravel()
    first = int(rng.integers(m))
    centres = [x[first].toarray().ravel()]
    d2 = np.maximum(x_sq + centres[0] @ centres[0] - 2.0 * (x @ centres[0]), 0.0)
    while len(centres) < k:
        tot = d2.sum()
        i = int(rng.integers(m)) if not tot > 0 else int(rng.choice(m, p=d2 / tot))
        c = x[i].toarray().ravel()
        centres.append(c)
        d2 = np.minimum(d2, np.maximum(x_sq + c @ c - 2.0 * (x @ c), 0.0))
    return np.array(centres, dtype=np.float64)


class DeviceKMeans:
    """The two device passes of one Lloyd step over the resident code columns ``cols`` (int32 device
    tensors, one per target column) of ``n_rows`` rows."""

    def __init__(self, ctx, cols, feats, n_rows, device):
        import torch
        self.torch, self.ctx, self.cols, self.feats, self.n, self.device = torch, ctx, cols, feats, n_rows, device
        self.labels = torch.zeros(max(n_rows, 1), dtype=torch.int32, device=device)
        self.host_s = 0.0

    def assign(self, centres, split=None):
        torch = self.torch
        t0 = time.perf_counter()
        P, mu_sq = self.feats.p_table(centres)
        self.host_s += time.perf_counter() - t0
        d_p = torch.from_numpy(P).to(self.device)
        d_mu = torch.from_numpy(mu_sq).to(self.device)
        d_split = None if split is None else torch.from_numpy(np.asarray(split, dtype=np.int32)).to(self.device)
        self.ctx.kmeans_assign(self.cols, self.feats.dom, self.feats.p_off, self.n, d_p, d_mu, self.labels, d_split)

    def counts(self, n_labels, lo=0):
        """N_c = counts of (label, code slot of column c) for the labels in [lo, n_labels) -> list of int64
        [n_labels][dom_c + 1] (rows below lo are 0).  Columns whose table fits shared memory go through dr_cooc,
        up to 63 per call next to the label column; wider ones through dr_label_counts (global memory)."""
        torch = self.torch
        out = [None] * len(self.cols)
        dom = self.feats.dom
        narrow = [i for i in range(len(self.cols)) if (n_labels + 1) * (dom[i] + 1) <= 65535]
        for b0 in range(0, len(narrow), 63):
            part = narrow[b0:b0 + 63]
            doms = [n_labels] + [dom[i] for i in part]
            sizes = [(n_labels + 1) * (dom[i] + 1) for i in part]
            off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
            tab = torch.zeros(int(off[-1]), dtype=torch.int64, device=self.device)
            self.ctx.cooc([self.labels] + [self.cols[i] for i in part], doms, [0] * len(part),
                          list(range(1, len(part) + 1)), off, self.n, tab)
            h = tab.cpu().numpy()
            for q, i in enumerate(part):
                n_c = h[off[q]:off[q + 1]].reshape(n_labels + 1, dom[i] + 1)[1:].copy()
                n_c[:lo] = 0
                out[i] = n_c
        for i in range(len(self.cols)):
            if out[i] is None:
                tab = torch.zeros((n_labels - lo, dom[i] + 1), dtype=torch.int64, device=self.device)
                self.ctx.label_counts(self.labels, self.cols[i], dom[i], self.n, lo, n_labels, tab)
                n_c = np.zeros((n_labels, dom[i] + 1), dtype=np.int64)
                n_c[lo:] = tab.cpu().numpy()
                out[i] = n_c
        return out


def _sample_codes(cols, n_rows, rng):
    """Codes of the k-means++ sample: every row up to SAMPLE_ROWS rows, else SAMPLE_ROWS distinct rows."""
    import torch
    if n_rows <= SAMPLE_ROWS:
        return [c[:n_rows].cpu().numpy() for c in cols]
    rows = np.sort(rng.choice(n_rows, size=SAMPLE_ROWS, replace=False))
    idx = torch.from_numpy(rows).to(cols[0].device)
    return [c.index_select(0, idx).cpu().numpy() for c in cols]


def kmeans(dk, k, info=None):
    """Spark's KMeans (maxIter 20, tol 1e-4) from k-means++ over the seeded sample; the final labels are the
    assignment to the final centres.  -> labels (device int32, in ``dk.labels``)."""
    rng = np.random.default_rng(SEED)
    x = dk.feats.rows(_sample_codes(dk.cols, dk.n, rng))
    centres = kmeanspp(x, k, rng)
    if info is not None:
        info["init_centres"] = centres.copy()
    it = 0
    while it < MAX_ITER:
        dk.assign(centres)
        counts = dk.counts(k)
        t0 = time.perf_counter()
        new, _ = dk.feats.centres_from_counts(counts, centres)
        converged = bool(np.all(((new - centres) ** 2).sum(axis=1) <= TOL * TOL))
        dk.host_s += time.perf_counter() - t0
        centres = new
        it += 1
        if converged:
            break
    dk.assign(centres)
    if info is not None:
        info.update(iterations=it, centres=centres)
    return dk.labels


def split_noise(node, n_terms):
    return np.random.default_rng([SEED, int(node)]).random(n_terms)


def bisecting_kmeans(dk, k, hist, n_rows, info=None):
    """Spark's BisectingKMeans (minDivisibleClusterSize 1, maxIter 20 per split) -> (labels, leaf LUT):
    the device labels are node ids, ``lut[id]`` is the leaf's index 0..k-1 in tree order."""
    feats = dk.feats
    root = np.zeros((1, feats.n_terms), dtype=np.float64)
    for b, h in zip(feats.B, hist):
        root[0] += np.asarray(b.T @ np.asarray(h, dtype=np.float64))
    if n_rows:
        root /= float(n_rows)
    centres = root                       # row i = centre of node id i
    heap = [1]                           # Spark's node index of each id
    size = [n_rows]
    children = {}                        # id -> ids of its non-empty children
    active = [0]
    needed = k - 1
    levels = 0
    while active and needed > 0:
        divisible = [i for i in active if size[i] >= 2]
        if len(divisible) > needed:
            divisible = sorted(divisible, key=lambda i: (-size[i], heap[i]))[:needed]
        if not divisible:
            break
        divisible = sorted(divisible, key=lambda i: heap[i])
        n_ids = len(heap) + 2 * len(divisible)
        split = np.full(n_ids, -1, dtype=np.int32)
        grown = np.zeros((n_ids, feats.n_terms), dtype=np.float64)
        grown[:len(heap)] = centres
        pairs = []
        for i in divisible:
            a = len(heap)
            heap += [2 * heap[i], 2 * heap[i] + 1]
            size += [0, 0]
            level = 1e-4 * float(np.sqrt(centres[i] @ centres[i]))
            noise = split_noise(heap[i], feats.n_terms)
            grown[a] = centres[i] - level * noise
            grown[a + 1] = centres[i] + level * noise
            split[i] = split[a] = split[a + 1] = a
            pairs.append((i, a))
        centres = grown
        first_child = len(heap) - 2 * len(divisible)
        for _ in range(MAX_ITER):
            dk.assign(centres, split)
            counts = dk.counts(n_ids, first_child)      # only the children being split move
            t0 = time.perf_counter()
            new, _ = feats.centres_from_counts(counts, centres)
            for _, a in pairs:
                centres[a:a + 2] = new[a:a + 2]
            dk.host_s += time.perf_counter() - t0
        dk.assign(centres, split)
        n_j = dk.counts(n_ids, first_child)[0].sum(axis=1)
        active = []
        for i, a in pairs:
            size[a], size[a + 1] = int(n_j[a]), int(n_j[a + 1])
            children[i] = [j for j in (a, a + 1) if size[j] > 0]
            if len(children[i]) == 2:
                active += [a, a + 1]
                needed -= 1
        levels += 1
    lut = np.zeros(len(heap), dtype=np.int32)
    n_leaves, stack = 0, [0]
    while stack:                         # depth first, left child first: Spark's leaf order
        i = stack.pop()
        if i in children and children[i]:
            stack += children[i][::-1]
        else:
            lut[i] = n_leaves
            n_leaves += 1
    if info is not None:
        info.update(levels=levels, centres=centres, heap=list(heap), n_leaves=n_leaves)
    return dk.labels, lut
