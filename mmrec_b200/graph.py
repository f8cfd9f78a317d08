"""Graph builders feeding the propagation kernel: vectorised replacements of the reference's Python-dict /
scipy builders.  Host logic (numpy) for the one-off normalised adjacency, device code for what changes per epoch.

Reference code replaced (paths relative to the root of enoche/MMRec):
  * `get_norm_adj_mat`  -- src/models/freedom.py:102-126 (copy-pasted in bm3/lightgcn/layergcn/encoders):
    a Python dict with 2E tuple keys, infeasible at 10^8 edges;
  * `MGCN.get_adj_mat`  -- src/models/mgcn.py:109-144 (lil-matrix slicing, 128 s at clothing scale);
  * `pre_epoch_processing` / `_normalize_adj_m` / `get_edge_info` -- src/models/freedom.py:128-162;
  * `get_knn_adj_mat` -- src/models/freedom.py:79-100 and `build_knn_normalized_graph` -- src/utils/utils.py:165-183
    (init-time item-item graphs; SURVEY.md 8f f4: contraction and selection on the scoring kernels, `_knn`).
"""
from __future__ import annotations

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

    def sample(self, dropout: float):
        keep_len = int(self.edge_values.size(0) * (1.0 - dropout))
        keep_idx = torch.multinomial(self.edge_values, keep_len)
        return self.adj_from_keep(keep_idx), keep_idx


# ------------------------------------------------------------------------------------------------
# item-item kNN graphs (init time)
# ------------------------------------------------------------------------------------------------
def _knn(feat: torch.Tensor, k: int):
    """Cosine kNN of the item features (`sim = cn @ cn.T; torch.topk(sim, k)`, src/models/freedom.py:79-84,
    src/utils/utils.py:165-172) on the scoring kernels (SURVEY.md 8f f4): the contraction is `ops.score` -- the same
    `U I^T` as full_sort_predict with the normalised features on both sides (exact fp32 fmaf chains for F > 128) -- in row
    blocks bounded to 256 MiB of similarities, the selection is `ops.mask_topk` (radix select, ties -> lower index)."""
    cn = feat.div(torch.norm(feat, p=2, dim=-1, keepdim=True)).contiguous()
    n = cn.shape[0]
    vals, inds = [], []
    step = max(128, (256 << 20) // (4 * n))
    for s in range(0, n, step):
        sim = ops.score(cn[s:s + step], cn)
        v, i = ops.mask_topk(sim, None, k)
        vals.append(v); inds.append(i)
    return torch.cat(vals), torch.cat(inds)


def freedom_knn_coo(feat: torch.Tensor, k: int):
    """`freedom.py:79-100`: directed cosine kNN, every edge weighs pow(k + 1e-7, -0.5)^2 in fp32."""
    _, ind = _knn(feat, k)
    n = feat.shape[0]
    row = torch.arange(n, device=feat.device).unsqueeze(1).expand(-1, k).reshape(-1)
    col = ind.reshape(-1)
    deg = torch.zeros(n, dtype=torch.int64, device=feat.device).index_add_(0, row, torch.ones_like(row))
    rinv = torch.pow(1e-7 + deg, -0.5)
    return row, col, rinv[row] * rinv[col]


def build_freedom_mm_adj(v_feat, t_feat, k: int, image_weight: float) -> CSR:
    """`freedom.py:67-75`: w * image_adj + (1 - w) * text_adj; shared edges add (CSR build sums duplicates)."""
    parts = []
    if v_feat is not None:
        parts.append((freedom_knn_coo(v_feat, k), image_weight if t_feat is not None else None))
    if t_feat is not None:
        parts.append((freedom_knn_coo(t_feat, k), (1.0 - image_weight) if v_feat is not None else None))
    rows = torch.cat([p[0][0] for p in parts])
    cols = torch.cat([p[0][1] for p in parts])
    vals = torch.cat([p[0][2] if p[1] is None else p[1] * p[0][2] for p in parts])
    n = (v_feat if v_feat is not None else t_feat).shape[0]
    return CSR.from_coo(rows, cols, vals, n, n, sum_duplicates=True, symmetric=False)


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
