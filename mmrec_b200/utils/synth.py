"""Seeded synthetic Amazon-shaped interaction graphs (SURVEY.md Appendix C).

Parity tests and bench numbers need no downloaded dataset: they run on graphs
drawn here.  The on-disk layout written by
:func:`write_dataset` is exactly what the reference reads
(`src/utils/dataset.py:50-55` -- a TSV with the columns named in
`src/configs/dataset/baby.yaml:2-9` plus `x_label`; `image_feat.npy` /
`text_feat.npy` per `baby.yaml:12-13`, loaded at
`src/common/abstract_recommender.py:90-103`).
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np

# name -> (users, items, train interactions, embedding dim, feature dim)
SHAPES = {
    "tiny": (300, 120, 2000, 64, 128),
    "small": (2000, 700, 16000, 64, 256),
    "baby": (20000, 7000, 160000, 64, 4096),        # BASELINE.json configs[0], [1]
    "sports": (36000, 18000, 300000, 64, 4096),     # configs[2]
    "clothing": (40000, 23000, 280000, 64, 4096),   # configs[3]
    "xl": (2000000, 1000000, 50000000, 128, 4096),  # configs[4] (never with dense features)
    # one GPU's share of a configs[4]-shaped job for the weak-scaling run (x N items and edges at N GPUs: 1M items at N = 8),
    # d = 128, user table and item shard beyond the L2; fewer users / edges than configs[4] so that the synthetic graph is
    # drawn in under a minute per rank
    "xls": (250000, 125000, 2000000, 128, 4096),
}


@dataclass
class SynthGraph:
    n_users: int
    n_items: int
    user: np.ndarray     # int64 [E_total]
    item: np.ndarray     # int64 [E_total]
    label: np.ndarray    # int8  [E_total]  0 train / 1 valid / 2 test

    def split(self, which: int):
        m = self.label == which
        return self.user[m], self.item[m]

    @property
    def train(self):
        return self.split(0)


def zipf_items(rng: np.random.Generator, n_items: int, size: int, s: float = 0.8) -> np.ndarray:
    """Items with popularity p_i ~ (i+1)^-s, drawn by inverse-CDF lookup."""
    w = (np.arange(n_items, dtype=np.float64) + 1.0) ** (-s)
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    return np.minimum(np.searchsorted(cdf, rng.random(size)), n_items - 1).astype(np.int64)


def _dedup(u: np.ndarray, i: np.ndarray, n_items: int):
    key = u * np.int64(n_items) + i
    _, first = np.unique(key, return_index=True)
    first.sort()  # keep draw order
    return u[first], i[first], first


def make_graph(n_users: int, n_items: int, n_train: int, seed: int = 0) -> SynthGraph:
    """Appendix C: E_total = E/0.8 labelled 0.8/0.1/0.1, every node has train degree >= 1."""
    rng = np.random.default_rng(seed)
    e_total = int(round(n_train / 0.8))
    n_draw = int(1.05 * e_total)
    u = rng.integers(0, n_users, n_draw, dtype=np.int64)
    i = zipf_items(rng, n_items, n_draw)
    u, i, _ = _dedup(u, i, n_items)
    keep = max(e_total - n_users - n_items, 0)
    u, i = u[:keep], i[:keep]
    lab = rng.choice(np.array([0, 1, 2], dtype=np.int8), size=u.shape[0], p=[0.8, 0.1, 0.1])
    # one guaranteed train edge per user and per item
    uu = np.arange(n_users, dtype=np.int64)
    ui = zipf_items(rng, n_items, n_users)
    ii = np.arange(n_items, dtype=np.int64)
    iu = rng.integers(0, n_users, n_items, dtype=np.int64)
    u = np.concatenate([uu, iu, u])
    i = np.concatenate([ui, ii, i])
    lab = np.concatenate([np.zeros(n_users + n_items, np.int8), lab])
    u, i, first = _dedup(u, i, n_items)
    lab = lab[first]
    return SynthGraph(n_users, n_items, u, i, lab)


def make_features(n_items: int, dim: int, seed: int = 1):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n_items, dim), dtype=np.float32)
    t = rng.standard_normal((n_items, dim), dtype=np.float32)
    return v, t


def named(name: str, seed: int = 0) -> SynthGraph:
    u, i, e, _, _ = SHAPES[name]
    return make_graph(u, i, e, seed)


def write_dataset(root: str, name: str, g: SynthGraph, v_feat=None, t_feat=None,
                  uid_field: str = "userID", iid_field: str = "itemID") -> str:
    """Write `<root>/<name>/<name>.inter` (+ feature .npy files) in the reference's format."""
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, f"{name}.inter"), "w") as f:
        f.write(f"{uid_field}\t{iid_field}\tx_label\n")
        np.savetxt(f, np.stack([g.user, g.item, g.label.astype(np.int64)], 1), fmt="%d", delimiter="\t")
    if v_feat is not None:
        np.save(os.path.join(d, "image_feat.npy"), v_feat)
    if t_feat is not None:
        np.save(os.path.join(d, "text_feat.npy"), t_feat)
    return d


def user_graph_dict(g: SynthGraph, max_neighbours: int = 200, block: int = 1024) -> dict:
    """The `user_graph_dict` of `preprocessing/dualgnn-gen-u-u-matrix.py` for `g` (DualGNN's user-user graph), without its
    U(U-1)/2 Python set intersections and dense U x U matrix: per user, `[neighbours, counts]` of the users who share
    training items with it (`x_label == 0`, each (user, item) pair counted once), best first, at most `max_neighbours`.

    Counts are the binarised training matrix's co-occurrences R R^T, from scipy sparse products over `block` users at a
    time, with the diagonal excluded (the script only counts pairs of distinct users).  Each user's row is then handed to
    the script's own expression, `torch.topk` of the dense fp32 row with k = min(non-zeros, max_neighbours), so ties come
    out in the script's order.  The script's U is the number of distinct users in the whole file."""
    import scipy.sparse as sp
    import torch
    n_users = int(np.unique(g.user).size)
    u, i = g.train
    n_items = int(g.item.max()) + 1 if g.item.size else 0
    R = sp.csr_matrix((np.ones(u.size, dtype=np.int64), (u, i)), shape=(n_users, n_items))
    R.sum_duplicates()
    R.data[:] = 1
    Rt = R.T.tocsr()
    out = {}
    for lo in range(0, n_users, block):
        hi = min(n_users, lo + block)
        C = np.asarray((R[lo:hi] @ Rt).todense(), dtype=np.float32)
        C[np.arange(hi - lo), np.arange(lo, hi)] = 0.0
        T = torch.from_numpy(C)
        nz = np.count_nonzero(C, axis=1)
        for r in range(hi - lo):
            top = torch.topk(T[r], int(min(nz[r], max_neighbours)))
            out[lo + r] = [top.indices.numpy().tolist(), top.values.numpy().tolist()]
    return out


def write_user_graph_dict(root: str, name: str, g: SynthGraph, file_name: str = "user_graph_dict.npy", **kw) -> str:
    """Write `<root>/<name>/<file_name>` (`user_graph_dict_file` of the dataset yaml) as the reference's preprocessing
    script does: `np.save` of the pickled dict of `user_graph_dict(g)`."""
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, file_name)
    np.save(path, user_graph_dict(g, **kw), allow_pickle=True)
    return path
