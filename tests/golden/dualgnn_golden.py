"""Shared by DualGNN's golden generator (make_golden_dualgnn.py) and its tests: the recorded graphs, the seeds, the
`user_graph_dict` as flat arrays (`ptr` [U + 1], `idx`, `val`: user u's neighbours are idx[ptr[u]:ptr[u + 1]]), and how a
recorded tensor is kept.

A tensor is kept as the SHA-256 of its bytes (`<key>.sha256`: bit equality) and, for comparisons within a tolerance,
either whole (`<key>`: up to SMALL elements, or where the file names it so) or as a sketch (`<key>.sketch`): its rows
times a fixed Gaussian matrix of SKETCH_COLS columns, computed in float64 and stored as fp32.  A random projection keeps
the norm of a difference to within a small factor, so the relative error of the sketches stands for the relative error of
the tensors, and a [256, 128] gradient takes 16 KiB instead of 128 KiB of incompressible bytes."""
import hashlib

import numpy as np

# synth.make_graph(users, items, train interactions, seed) of the two graphs the preprocessing script was run on:
# `tiny` (the model's dataset) and a small dense one where most co-occurrence counts tie
GRAPHS = {"tiny": None, "ties": (90, 12, 420, 3)}
SAMPLE_SEED = 2024            # np.random.seed before the recorded `pre_epoch_processing`
BATCH_SEED = 7
EPOCH_SEED0 = 3000            # np.random.seed(EPOCH_SEED0 + epoch) before each trajectory epoch's `pre_epoch_processing`
K = 40


def sha256(a) -> str:
    """SHA-256 of the array's bytes in its own dtype (float64 stays float64)."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.dtype.str.encode() + a.tobytes()).hexdigest()


SMALL = 4096
SKETCH_COLS = 16


def sketch(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    a = a.reshape(a.shape[0], -1)
    R = np.random.default_rng(a.shape[1]).standard_normal((a.shape[1], SKETCH_COLS))
    return (a @ R).astype(np.float32)


def put_sha(g: dict, key: str, a):
    g[key + ".sha256"] = np.array(sha256(a))


def put(g: dict, key: str, a, whole: bool = False):
    """Record `a` under `key`: its digest, and the tensor itself or its sketch."""
    a = np.asarray(a)
    put_sha(g, key, a)
    if whole or a.size <= SMALL:
        g[key] = a.copy()
    else:
        g[key + ".sketch"] = sketch(a)


def equal(gold, key, a) -> bool:
    """`a` has the recorded bits (dtype and shape included)."""
    return sha256(np.asarray(a)) == str(gold[key + ".sha256"])


def rel(gold, key, a) -> float:
    """Relative 2-norm difference of `a` from the recorded tensor, or of their sketches."""
    a = np.asarray(a, dtype=np.float64)
    if key in gold:
        ref, got = np.asarray(gold[key], dtype=np.float64), a
    else:
        ref, got = np.asarray(gold[key + ".sketch"], dtype=np.float64), sketch(a)
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))


def recorded(gold, prefix: str) -> list:
    """The keys recorded under `prefix` (e.g. "grad."), without the `.sha256` / `.sketch` suffixes."""
    keys = {str(k) for k in (gold.files if hasattr(gold, "files") else gold)}
    return sorted({k[:-len(".sha256")] for k in keys if k.startswith(prefix) and k.endswith(".sha256")})


def flatten(d: dict):
    n = len(d)
    lens = np.array([len(d[u][0]) for u in range(n)], dtype=np.int64)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.array([j for u in range(n) for j in d[u][0]], dtype=np.int64)
    val = np.array([w for u in range(n) for w in d[u][1]], dtype=np.float64)
    return ptr, idx, val


def topk_sample_loop(user_graph_dict, k, rng=np.random):
    """The reference's `topk_sample` loop (`src/models/dualgnn.py:207-250`, softmax mode) restated with its scalar draws:
    the yardstick of the vectorised sampler."""
    import torch
    import torch.nn.functional as F
    index, weights = [], torch.zeros(len(user_graph_dict), k)
    for i in range(len(user_graph_dict)):
        nb, wt = user_graph_dict[i][0], user_graph_dict[i][1]
        if len(nb) < k:
            if len(nb) == 0:
                index.append([0] * k)
                continue
            s, w = list(nb[:k]), list(wt[:k])
            while len(s) < k:
                r = rng.randint(0, len(s))
                s.append(s[r])
                w.append(w[r])
            index.append(s)
            weights[i] = F.softmax(torch.tensor(w), dim=0)
            continue
        index.append(list(nb[:k]))
        weights[i] = F.softmax(torch.tensor(list(wt[:k])), dim=0)
    return np.array(index, dtype=np.int64), weights.numpy()
