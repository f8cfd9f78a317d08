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
