"""Shared by DualGNN's golden generator (make_golden_dualgnn.py) and its tests: the recorded graphs, the seeds, and the
`user_graph_dict` as flat arrays (`ptr` [U + 1], `idx`, `val`: user u's neighbours are idx[ptr[u]:ptr[u + 1]]).  How a
recorded tensor is kept: golden_io.py."""
import numpy as np

# synth.make_graph(users, items, train interactions, seed) of the two graphs the preprocessing script was run on:
# `tiny` (the model's dataset) and a small dense one where most co-occurrence counts tie
GRAPHS = {"tiny": None, "ties": (90, 12, 420, 3)}
SAMPLE_SEED = 2024            # np.random.seed before the recorded `pre_epoch_processing`
BATCH_SEED = 7
EPOCH_SEED0 = 3000            # np.random.seed(EPOCH_SEED0 + epoch) before each trajectory epoch's `pre_epoch_processing`
K = 40


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
