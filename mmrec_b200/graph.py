"""Graph builders feeding the propagation kernel: vectorised replacements of the reference's Python-dict /
scipy builders.  Host logic (numpy) for the one-off normalised adjacency, device code for what changes per epoch.

Reference code replaced (paths relative to the root of enoche/MMRec):
  * `get_norm_adj_mat`  -- src/models/freedom.py:102-126 (copy-pasted in bm3/lightgcn/layergcn/encoders):
    a Python dict with 2E tuple keys, infeasible at 10^8 edges;
  * `MGCN.get_adj_mat`  -- src/models/mgcn.py:109-144 (lil-matrix slicing, 128 s at clothing scale);
  * `pre_epoch_processing` / `_normalize_adj_m` / `get_edge_info` -- src/models/freedom.py:128-162;
  * `get_knn_adj_mat` -- src/models/freedom.py:79-100 and `build_knn_normalized_graph` -- src/utils/utils.py:165-183
    (init-time item-item graphs; SURVEY.md 8f f4: contraction and selection on the scoring kernels, `_knn`);
  * `get_adj_mat` -- src/models/lattice.py:100-122 (LATTICE's D^-1 (A + I) through dok / lil): `lattice_norm_adj_entries`;
  * `build_sim` / `build_knn_neighbourhood` / `compute_normalized_laplacian` -- src/utils/utils.py:119-137 (LATTICE's
    dense [I, I] graphs): `build_mgcn_knn_adj` at construction, `knn_normalized` for the learned graph.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops
from .ops import CSR


def unique_sorted(keys: np.ndarray) -> np.ndarray:
    """`np.unique(keys)` for large integer arrays as sort + neighbour compare: the same values in the same order, but ~100x
    faster than numpy 2.3's `unique` at 10^6..10^8 keys (4 M keys: 0.07 s against 5.7 s; the 10^8 keys of a config-5 graph:
    seconds against ten minutes) -- the adjacency build is the part of the reference that cannot scale (freedom.py:102-111)."""
    if keys.size == 0:
        return keys.copy()
    s = np.sort(keys, kind="stable")
    keep = np.empty(s.size, dtype=bool)
    keep[0] = True
    np.not_equal(s[1:], s[:-1], out=keep[1:])
    return s[keep]


def _sym_keys(inter_row, inter_col, n_users, n_items):
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    n = n_users + n_items
    key = unique_sorted(np.concatenate([r * n + (c + n_users), (c + n_users) * n + r]))   # binary, de-duplicated
    return key // n, key % n, n


def norm_adj_entries(inter_row, inter_col, n_users, n_items):
    """(rows, cols, vals fp32) of D^-1/2 A D^-1/2: degrees + 1e-7 and both scalings in float64, rounded to fp32
    once, exactly as `freedom.py:113-124` does through scipy."""
    rows, cols, n = _sym_keys(inter_row, inter_col, n_users, n_items)
    deg = np.bincount(rows, minlength=n).astype(np.float64) + 1e-7
    dinv = np.power(deg, -0.5)
    vals = ((dinv[rows] * 1.0) * dinv[cols]).astype(np.float32)
    return rows, cols, vals


def mgcn_norm_adj_entries(inter_row, inter_col, n_users, n_items):
    """MGCN's normalisation (`mgcn.py:118-129`): float32 throughout, no epsilon, inf -> 0."""
    rows, cols, n = _sym_keys(inter_row, inter_col, n_users, n_items)
    rowsum = np.bincount(rows, minlength=n).astype(np.float32)
    with np.errstate(divide="ignore"):
        dinv = np.power(rowsum, np.float32(-0.5)).astype(np.float32)
    dinv[np.isinf(dinv)] = 0.0
    vals = ((dinv[rows] * np.float32(1.0)).astype(np.float32) * dinv[cols]).astype(np.float32)
    return rows, cols, vals


SLMREC_SYMMETRIC_ADJ = ("plain", "pre")


def slmrec_adj_entries(inter_row, inter_col, n_users, n_items, adj_type):
    """(rows, cols, vals fp32) of SLMRec's `create_adj_mat` (`src/models/slmrec.py:434-479`) for each `adj_type`, with the
    dtypes its scipy calls compute in, so that the values equal the fp32 ones it hands to `torch.sparse.FloatTensor`:

    * `plain`: the binary symmetric A (float32 ones);
    * `norm`: D^-1 (A + I) -- `sp.eye` is float64, so the degrees + 1 and `np.power(., -1)` are float64, rounded to fp32 once;
    * `gcmc`: D^-1 A in float32 (`np.power(deg, -1)` of the float32 degrees, inf -> 0);
    * `pre`: D^-1/2 A D^-1/2 in float32: `deg + 1e-08` and `np.power(., -0.5)` in float32, one fp32 product per entry;
    * anything else (`mean`): the float32 D^-1 A of `gcmc` plus I, the diagonal 1.0.

    Only `plain` and `pre` are symmetric (SLMREC_SYMMETRIC_ADJ).  Entries in (row, col) order."""
    rows, cols, n = _sym_keys(inter_row, inter_col, n_users, n_items)
    deg = np.bincount(rows, minlength=n)
    if adj_type == "plain":
        return rows, cols, np.ones(rows.size, dtype=np.float32)
    if adj_type == "pre":
        with np.errstate(divide="ignore"):
            dinv = np.power(deg.astype(np.float32) + 1e-08, -0.5)
        dinv[np.isinf(dinv)] = 0.0
        return rows, cols, (dinv[rows] * dinv[cols]).astype(np.float32)
    if adj_type == "norm":
        dinv = np.power(deg.astype(np.float64) + 1.0, -1)
        diag = np.arange(n, dtype=np.int64)
        key = np.concatenate([rows * n + cols, diag * n + diag])
        order = np.argsort(key, kind="stable")
        r, c = key[order] // n, key[order] % n
        return r, c, dinv[r].astype(np.float32)
    with np.errstate(divide="ignore"):
        dinv = np.power(deg.astype(np.float32), -1)
    dinv[np.isinf(dinv)] = 0.0
    if adj_type == "gcmc":
        return rows, cols, dinv[rows].astype(np.float32)
    diag = np.arange(n, dtype=np.int64)                               # mean: D^-1 A + I (bipartite: no diagonal in D^-1 A)
    key = np.concatenate([rows * n + cols, diag * n + diag])
    vals = np.concatenate([dinv[rows].astype(np.float32), np.ones(n, dtype=np.float32)])
    order = np.argsort(key, kind="stable")
    return key[order] // n, key[order] % n, vals[order]


def build_slmrec_adj(inter, n_users, n_items, device, adj_type) -> CSR:
    """SLMRec's `norm_adj` (`slmrec.py:40-44`) as a device CSR; flagged symmetric for `plain` and `pre` only, so the
    others take their backward on `CSR.t()`."""
    r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
    rows, cols, vals = slmrec_adj_entries(r, c, n_users, n_items, adj_type)
    n = n_users + n_items
    return CSR.from_coo(_to_dev(rows, device), _to_dev(cols, device), _to_dev(vals, device), n, n,
                        sum_duplicates=False, symmetric=adj_type in SLMREC_SYMMETRIC_ADJ)


def lattice_norm_adj_entries(inter_row, inter_col, n_users, n_items):
    """(rows, cols, vals fp32) of LATTICE's `get_adj_mat` (`src/models/lattice.py:100-122`): D^-1 (A + I), row-normalised
    with self-loops.  The reference assigns R into a lil matrix, so a repeated (user, item) pair keeps its multiplicity m
    as the entry's value (SLMRec's `nonzero()` makes it binary, `slmrec_adj_entries`); `sp.eye` is float64, so the row sums
    and `np.power(rowsum, -1)` are float64 and each value is fl32(d_inv[r] * m), rounded once.  Entries in (row, col)
    order; no dok or lil matrix is built."""
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    n = n_users + n_items
    diag = np.arange(n, dtype=np.int64)
    key = np.sort(np.concatenate([r * n + (c + n_users), (c + n_users) * n + r, diag * n + diag]), kind="stable")
    start = np.empty(key.size, dtype=bool)
    start[0] = True                                                   # n >= 1: the diagonal is never empty
    np.not_equal(key[1:], key[:-1], out=start[1:])
    first = np.flatnonzero(start)
    mult = np.diff(np.append(first, key.size)).astype(np.float64)
    ukey = key[first]
    rows, cols = ukey // n, ukey % n
    d_inv = np.power(np.bincount(rows, weights=mult, minlength=n), -1)
    return rows, cols, (d_inv[rows] * mult).astype(np.float32)


def build_lattice_norm_adj(inter, n_users, n_items, device) -> CSR:
    """LATTICE's `norm_adj` as a device CSR, with its transpose (the backward's: the matrix is not symmetric)."""
    r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
    rows, cols, vals = lattice_norm_adj_entries(r, c, n_users, n_items)
    n = n_users + n_items
    A = CSR.from_coo(_to_dev(rows, device), _to_dev(cols, device), _to_dev(vals, device), n, n, sum_duplicates=False, symmetric=False)
    A.t()
    return A


def dropout_entry_maps(inter_row, inter_col, n_users, n_items):
    """The two index maps of SelfCF's per-batch edge dropout on `build_norm_adj`'s CSR (`src/common/encoders.py:77-88`):

    * `draw_of` int32[nnz]: draw j of `torch.rand(nnz)` belongs to the reference's j-th stored entry of `sparse_norm_adj`,
      which is CSR position e with draw_of[e] = j;
    * `mirror` int32[nnz]: the CSR position of (c, r) for the entry (r, c) at position e (the matrix is symmetric, so the
      dropped matrix's transpose is the same CSR with the keep bits read through `mirror`).

    The reference's stored order is that of `sp.coo_matrix(D * A * D)` with `A` the dok built from a dict
    (`encoders.py:51-70`).  With the scipy of this image (1.18) that order is: rows ascending, and within a row the
    first-insertion order of the dict -- the interaction COO's (u, i + n_users) pairs, then its (i + n_users, u) pairs, a
    repeated pair at its first position.  (Measured; it is the order of `A.tocsr()`.  Another scipy may store the product
    differently: the masks then match in distribution only.)  So the order is a stable sort by row of the de-duplicated
    concatenation, and each of its keys is found in the sorted keys of the CSR; no dok or scipy product is built."""
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    n = n_users + n_items
    key = np.concatenate([r * n + (c + n_users), (c + n_users) * n + r])
    order = np.argsort(key, kind="stable")                           # equal keys keep their order: the first occurrence leads
    s = key[order]
    start = np.empty(s.size, dtype=bool)
    if s.size:
        start[0] = True
        np.not_equal(s[1:], s[:-1], out=start[1:])
    ukey = s[start]                                                   # = the CSR's (row, col) keys in CSR order
    first = order[start]                                              # first position of each key in the concatenation
    ref = np.lexsort((first, ukey // n))                             # CSR positions in the reference's stored order
    draw_of = np.empty(ukey.size, dtype=np.int32)
    draw_of[ref] = np.arange(ukey.size, dtype=np.int32)
    mirror = np.searchsorted(ukey, (ukey % n) * n + ukey // n).astype(np.int32)
    return draw_of, mirror


def grcn_edge_order(inter_row, inter_col, n_users, n_items):
    """(rows, cols, order) of GRCN's attention graph (`src/models/grcn.py:158-159, 191-193`): the reference's symmetric edge
    list `cat(edge_index, edge_index[[1, 0]])` with `edge_index` = the interaction COO's (u, i + n_users) pairs, edge k going
    from source `src[k]` to target `dst[k]`, as a CSR over the targets.  Every interaction stays its own entry, as PyG sees
    it.  CSR position e holds the reference's edge `order[e]`: a stable sort by (target, source), so repeated edges keep
    their order.  rows = dst[order], cols = src[order] (the source node, whose `model_specific_conf` row weights the edge)."""
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64) + n_users
    n = n_users + n_items
    src, dst = np.concatenate([r, c]), np.concatenate([c, r])
    order = np.argsort(dst * n + src, kind="stable")
    return dst[order], src[order], order


def build_grcn_adj(inter, n_users, n_items, device):
    """(CSR, order int64 on the device) of `grcn_edge_order`.  The CSR build's sort is stable and the entries arrive sorted,
    so its stored order is the host order.  Its transpose pattern and heavy-row list are built here too, so that a step can
    be captured in a CUDA graph."""
    r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
    rows, cols, order = grcn_edge_order(r, c, n_users, n_items)
    n = n_users + n_items
    A = CSR.from_coo(_to_dev(rows, device), _to_dev(cols, device), None, n, n, sum_duplicates=False, symmetric=False)
    A.transpose_pattern()
    ops.edge_attention_heavy_rows(A)
    return A, _to_dev(order, device)


def _to_dev(a, device, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(device=device, dtype=dtype) if dtype is not None else t.to(device)


def build_norm_adj(inter, n_users, n_items, device, variant="lightgcn") -> CSR:
    """Normalised (U+I) x (U+I) adjacency as a device CSR.  `inter` is the scipy COO from
    `dataloader.inter_matrix(form='coo')` or an (row, col) pair."""
    r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
    fn = mgcn_norm_adj_entries if variant == "mgcn" else norm_adj_entries
    rows, cols, vals = fn(r, c, n_users, n_items)
    n = n_users + n_items
    return CSR.from_coo(_to_dev(rows, device), _to_dev(cols, device), _to_dev(vals, device), n, n,
                        sum_duplicates=False, symmetric=True)


def gcn_add_entries(edge_index: torch.Tensor, n_nodes: int):
    """(dst, src, norm fp32) of DualGNN's `Base_gcn` with `aggr='add'` (`src/models/dualgnn.py:325-341`), PyG's `gcn`-style
    norm: `remove_self_loops`, `deg = degree(row)` (an fp32 `index_add` of ones), `deg.pow(-0.5)`, `norm = dis[row] *
    dis[col]`, and the message `norm * x[row]` summed at `col`.  The same fp32 torch expressions on the host, so the values
    equal the reference's bit for bit.  No epsilon: unlike `norm_adj_entries` a node of degree 0 has no entries to scale."""
    ei = edge_index.detach().to("cpu", torch.int64)
    ei = ei[:, ei[0] != ei[1]]
    row, col = ei[0], ei[1]
    deg = torch.zeros(n_nodes, dtype=torch.float32).index_add_(0, row, torch.ones(row.numel(), dtype=torch.float32))
    dis = deg.pow(-0.5)
    return col, row, dis[row] * dis[col]


def build_gcn_add_adj(edge_index: torch.Tensor, n_nodes: int, device) -> CSR:
    """`gcn_add_entries` as a device CSR.  Repeated edges stay separate terms, as in the reference's scatter.  The edge list
    must hold both directions of every edge (DualGNN's, `dualgnn.py:59-60`): the matrix is then symmetric bit for bit
    (dis[r] * dis[c] == dis[c] * dis[r]) and its backward reads the same CSR."""
    dst, src, val = gcn_add_entries(edge_index, n_nodes)
    return CSR.from_coo(dst.to(device), src.to(device), val.to(device), n_nodes, n_nodes, sum_duplicates=False, symmetric=True)


class UserGraphTable:
    """DualGNN's `user_graph_dict` (`{user: [neighbours, co-occurrence counts]}`, at most 200 per user, best first; written
    by `preprocessing/dualgnn-gen-u-u-matrix.py` or `synth.write_user_graph_dict`) as arrays, converted once: the first
    min(n_u, k) neighbours `idx` int64 [U, k] and their counts `w` fp32 [U, k] (zero-padded), and `n` = min(n_u, k)."""

    def __init__(self, user_graph_dict: dict, k: int):
        n_users = len(user_graph_dict)
        self.k = k
        self.idx = np.zeros((n_users, k), dtype=np.int64)
        self.w = np.zeros((n_users, k), dtype=np.float32)
        self.n = np.zeros(n_users, dtype=np.int64)
        for u in range(n_users):                                      # the dict's keys are 0 .. U-1, as the script writes them
            nb, wt = user_graph_dict[u][0][:k], user_graph_dict[u][1][:k]
            m = len(nb)
            self.n[u] = m
            if m:
                self.idx[u, :m] = nb
                self.w[u, :m] = np.asarray(wt, dtype=np.float64).astype(np.float32)   # torch.tensor(list of floats): fp32

    def sample(self, rng=np.random):
        """`DualGNN.topk_sample(k)` (`dualgnn.py:207-250`) with `user_aggr_mode = 'softmax'`: (index int64 [U, k], weights fp32
        [U, k]).  A user with 0 < n_u < k neighbours is padded by `sample.append(sample[randint(0, len(sample))])`, the bound
        growing with each append; the draws come from `rng` (the reference's global `np.random`) in the reference's order,
        users ascending and appends in turn, as one `randint` call with an array of bounds: the same stream as the
        reference's scalar calls (tests/test_dualgnn_host.py).  Rows are then softmax-ed as one [U', k] fp32 tensor, the
        same bits as the reference's per-row `F.softmax(torch.tensor(weights), dim=0)` (also tested).  A user with no
        neighbours keeps the reference's row of index 0 with weight 0."""
        k = self.k
        idx, w = self.idx.copy(), self.w.copy()
        pos = np.arange(k)
        short = (self.n > 0) & (self.n < k)
        pad = short[:, None] & (pos[None, :] >= self.n[:, None])    # the appended slots, row-major = the reference's draw order
        users, slots = np.nonzero(pad)
        if users.size:
            draws_2d = np.zeros_like(idx)
            draws_2d[users, slots] = rng.randint(0, slots)            # bound = len(sample) at the append = the slot
            for p in range(int(self.n[short].min()), k):              # slot p copies an earlier slot, possibly itself a copy
                rows = users[slots == p]
                src = draws_2d[rows, p]
                idx[rows, p] = idx[rows, src]
                w[rows, p] = w[rows, src]
        weights = np.zeros((idx.shape[0], k), dtype=np.float32)
        have = self.n > 0
        if have.any():
            weights[have] = torch.softmax(torch.from_numpy(w[have]), dim=1).numpy()
        return idx, weights


def build_user_graph(idx: np.ndarray, weights: np.ndarray, device) -> CSR:
    """The per-epoch user graph G [U, U]: G[u, idx[u, j]] += weights[u, j], so that `G @ X` is `User_Graph_sample`'s
    `matmul(weights.unsqueeze(1), X[idx]).squeeze()` (`dualgnn.py:259-266`) without the [U, k, d] gather.  Repeated
    neighbours (the padding) stay separate terms (`sum_duplicates=False`), as in the reference's product.  Users without
    neighbours (weights 0) get no entries.  The transpose, which the backward reads, is built here too."""
    n_users, k = idx.shape
    keep = np.repeat(weights.any(axis=1), k)
    rows = np.repeat(np.arange(n_users, dtype=np.int64), k)[keep]
    G = CSR.from_coo(_to_dev(rows, device), _to_dev(idx.reshape(-1)[keep], device), _to_dev(weights.reshape(-1)[keep], device),
                     n_users, n_users, sum_duplicates=False, symmetric=False)
    G.t()
    return G


def build_mgcn_R(inter, n_users, n_items, device) -> CSR:
    """`self.R` = the U x I block of MGCN's normalised matrix (`mgcn.py:134`)."""
    r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
    rows, cols, vals = mgcn_norm_adj_entries(r, c, n_users, n_items)
    m = rows < n_users
    return CSR.from_coo(_to_dev(rows[m], device), _to_dev(cols[m] - n_users, device), _to_dev(vals[m], device),
                        n_users, n_items, sum_duplicates=False, symmetric=False)


class EdgePruner:
    """Degree-sensitive edge pruning of FREEDOM / LayerGCN (`freedom.py:128-162`, `layergcn.py:51-89`).

    The draw stays `torch.multinomial(edge_values, keep_len)` on the device tensor -- the same call on the same
    weights; everything after the draw (degree recount, renormalisation, symmetrisation, CSR build) runs in this
    library's kernels once per epoch.

    Edge order: sorted, de-duplicated (user, item) pairs.  That is what the reference's `get_edge_info` yields with the
    scipy of this image (`astype` canonicalises the COO matrix; `tests/golden/freedom_tiny.npz:edge_indices`, checked
    bit for bit), so the same seed prunes the same edges here.  An older scipy keeps the file's row order and repeated
    interactions: there the pruning matches in distribution only, and a repeated (u, i) counts once in the degrees.
    """

    def __init__(self, inter, n_users, n_items, device):
        r, c = (inter.row, inter.col) if hasattr(inter, "row") else inter
        r, c = np.asarray(r, dtype=np.int64), np.asarray(c, dtype=np.int64)
        key = unique_sorted(r * n_items + c)  # canonical (user, item) order, see oracle.edge_info
        self.n_users, self.n_items = n_users, n_items
        self.edge_indices = _to_dev(np.stack([key // n_items, key % n_items]), device)
        self.edge_values = ops.bipartite_norm(self.edge_indices[0], self.edge_indices[1], n_users, n_items)

    def adj_from_keep(self, keep_idx: torch.Tensor) -> CSR:
        keep = self.edge_indices[:, keep_idx]
        u, i = keep[0], keep[1]
        vals = ops.bipartite_norm(u, i, self.n_users, self.n_items)
        iu = i + self.n_users
        n = self.n_users + self.n_items
        return CSR.from_coo(torch.cat((u, iu)), torch.cat((iu, u)), torch.cat((vals, vals)), n, n,
                            sum_duplicates=True, symmetric=True)

    def sample(self, dropout: Optional[float] = None, keep_len: Optional[int] = None):
        """The epoch's pruned graph and the kept edges: `keep_len` edges (default `int(nnz * (1 - dropout))`, FREEDOM's;
        PGL's `int(nnz * 0.3)` is given as is, as the float product can round differently) drawn without replacement."""
        if keep_len is None:
            keep_len = int(self.edge_values.size(0) * (1.0 - dropout))
        keep_idx = torch.multinomial(self.edge_values, keep_len)
        return self.adj_from_keep(keep_idx), keep_idx


# ------------------------------------------------------------------------------------------------
# item-item kNN graphs (init time)
# ------------------------------------------------------------------------------------------------
def _knn(feat: torch.Tensor, k: int, rows: Optional[torch.Tensor] = None):
    """Cosine kNN of the item features (`sim = cn @ cn.T; torch.topk(sim, k)`, src/models/freedom.py:79-84,
    src/utils/utils.py:165-172), for the query rows `rows` (default: all), ties -> lower index (SURVEY.md 8f f4).

    F > 128 (every real feature table): `ops.knn_topk` (K7, csrc/knn_cf.cu) -- tensor-core candidate filter with the top-k
    fused and every value an exact fp32 fmaf chain, bit-identical to the route below at these widths (where `ops.score`
    is the exact CUDA-core kernel) without writing the [n, n] similarities.  F <= 128: `ops.score` (3xTF32 tensor-core
    path) in row blocks bounded to 256 MiB of similarities, then `ops.mask_topk` (radix select)."""
    return knn_normalized(feat.div(torch.norm(feat, p=2, dim=-1, keepdim=True)).contiguous(), k, rows)


def knn_normalized(cn: torch.Tensor, k: int, rows: Optional[torch.Tensor] = None):
    """`_knn` of features already divided by their row norms: (values, indices) [n_rows, k] of `cn @ cn.T`, no [n, n]
    tensor beyond the bounded score blocks.  LATTICE's learned graph selects on its own normalised projections."""
    cn = cn.contiguous()
    if cn.shape[1] > 128:
        return ops.knn_topk(cn, k, rows)
    n = cn.shape[0]
    q = cn if rows is None else cn.index_select(0, rows.to(device=cn.device, dtype=torch.int64))
    vals, inds = [], []
    step = max(128, (256 << 20) // (4 * n))
    for s in range(0, q.shape[0], step):
        sim = ops.score(q[s:s + step], cn)
        v, i = ops.mask_topk(sim, None, k)
        vals.append(v); inds.append(i)
    return torch.cat(vals), torch.cat(inds)


def freedom_knn_coo(feat: torch.Tensor, k: int, rows: Optional[torch.Tensor] = None):
    """`freedom.py:79-100`: directed cosine kNN, every edge weighs pow(k + 1e-7, -0.5)^2 in fp32.  `rows`: only the
    edges leaving those items (row ids stay global).  Every item has exactly k out-edges, so the degree of every item is k
    whichever rows are built: the rows are independent."""
    _, ind = _knn(feat, k, rows)
    n = feat.shape[0]
    src = torch.arange(n, device=feat.device) if rows is None else rows.to(device=feat.device, dtype=torch.int64)
    row = src.unsqueeze(1).expand(-1, k).reshape(-1)
    col = ind.reshape(-1)
    if rows is None:
        deg = torch.zeros(n, dtype=torch.int64, device=feat.device).index_add_(0, row, torch.ones_like(row))
    else:
        deg = torch.full((n,), k, dtype=torch.int64, device=feat.device)
    rinv = torch.pow(1e-7 + deg, -0.5)
    return row, col, rinv[row] * rinv[col]


def freedom_mm_entries(v_feat, t_feat, k: int, image_weight: float, rows: Optional[torch.Tensor] = None):
    """COO entries (pos, col, val) of `freedom.py:67-75`'s w * image_adj + (1 - w) * text_adj, image entries first, for
    the rows `rows` (default: all): `pos` = j for an entry of row rows[j].  Shared edges are not yet summed."""
    parts = []
    if v_feat is not None:
        parts.append((freedom_knn_coo(v_feat, k, rows), image_weight if t_feat is not None else None))
    if t_feat is not None:
        parts.append((freedom_knn_coo(t_feat, k, rows), (1.0 - image_weight) if v_feat is not None else None))
    n = (v_feat if v_feat is not None else t_feat).shape[0]
    if rows is None:
        pos = torch.cat([p[0][0] for p in parts])
    else:
        own = torch.arange(rows.numel(), device=parts[0][0][0].device).unsqueeze(1).expand(-1, k).reshape(-1)
        pos = torch.cat([own] * len(parts))
    cols = torch.cat([p[0][1] for p in parts])
    vals = torch.cat([p[0][2] if p[1] is None else p[1] * p[0][2] for p in parts])
    return pos, cols, vals, n


def build_freedom_mm_adj(v_feat, t_feat, k: int, image_weight: float, rows: Optional[torch.Tensor] = None) -> CSR:
    """`freedom.py:67-75`: w * image_adj + (1 - w) * text_adj; shared edges add (CSR build sums duplicates).  `rows`: the
    [len(rows), n] matrix whose row j is row rows[j] of mm_adj (FREEDOM's rows are independent, see freedom_knn_coo)."""
    pos, cols, vals, n = freedom_mm_entries(v_feat, t_feat, k, image_weight, rows)
    m = n if rows is None else rows.numel()
    return CSR.from_coo(pos, cols, vals, m, n, sum_duplicates=True, symmetric=False)


def build_mgcn_knn_adj(feat: torch.Tensor, k: int) -> CSR:
    """`utils.py:165-183` with `get_sparse_laplacian(normalization='sym')` (`:134-148`): cosine-weighted kNN."""
    val, ind = _knn(feat, k)
    n = feat.shape[0]
    row = torch.arange(n, device=feat.device).unsqueeze(1).expand(-1, k).reshape(-1)
    col = ind.reshape(-1)
    w = val.reshape(-1)
    deg = torch.zeros(n, dtype=w.dtype, device=w.device).index_add_(0, row, w)
    dis = deg.pow(-0.5)
    dis.masked_fill_(dis == float("inf"), 0)
    return CSR.from_coo(row, col, dis[row] * w * dis[col], n, n, sum_duplicates=True, symmetric=False)
