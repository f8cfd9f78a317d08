"""DualGNN's host-side pieces without a GPU: the user-graph file, the per-epoch sampler, the 'add' adjacency's values and
the refused configurations.

- `synth.write_user_graph_dict` writes what the reference's preprocessing script wrote (tests/golden/dualgnn_tiny.npz,
  make_golden_dualgnn.py) on `tiny` and on a small graph where most counts tie, neighbour order included.
- `graph.UserGraphTable.sample` equals the recorded `topk_sample` of the reference's class, and a restatement of its loop
  with scalar `np.random.randint` draws: the same index, weights and generator state after, also with short and empty
  neighbour lists.
- `graph.gcn_add_entries` equals PyG's gcn-norm expression (`dualgnn.py:335-341`) bit for bit."""
import functools
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import dualgnn_golden as D  # noqa: E402
import golden_io as G  # noqa: E402
from mmrec_b200 import graph  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402


def _graph(name):
    return synth.named(name) if D.GRAPHS[name] is None else synth.make_graph(*D.GRAPHS[name])


@functools.lru_cache(maxsize=None)
def _dict(name):
    """The user graph of a recorded graph, as `write_user_graph_dict` writes it (pinned to the script's file below)."""
    return synth.user_graph_dict(_graph(name))


@pytest.mark.parametrize("name", list(D.GRAPHS))
def test_user_graph_dict_equals_the_script(golden, name):
    gold = golden("dualgnn_tiny.npz")
    path = synth.write_user_graph_dict(tempfile.mkdtemp(prefix="mmrec_ugd_"), name, _graph(name))
    d = np.load(path, allow_pickle=True).item()
    ptr, idx, val = D.flatten(d)
    assert G.equal(gold, "ugd_%s_ptr" % name, ptr)
    assert G.equal(gold, "ugd_%s_idx" % name, idx)
    assert G.equal(gold, "ugd_%s_val" % name, val)
    assert all(type(j) is int for j in d[0][0]) and all(type(w) is float for w in d[0][1])
    assert d == _dict(name)
    if name == "ties":                                                # the order within ties is what this graph pins
        assert int((val[1:] == val[:-1]).sum()) > len(val) // 2


def test_sampler_equals_the_reference(golden):
    gold = golden("dualgnn_tiny.npz")
    np.random.seed(D.SAMPLE_SEED)
    idx, w = graph.UserGraphTable(_dict("tiny"), D.K).sample(np.random)
    assert G.equal(gold, "sample_idx", idx) and G.equal(gold, "sample_w", w)


@pytest.mark.parametrize("name", list(D.GRAPHS))
@pytest.mark.parametrize("cut", [None, 7, 13])
def test_vectorised_draws_and_softmax_equal_the_loop(name, cut):
    """One `randint` with an array of bounds draws what the reference's scalar calls draw, and the batched softmax gives
    each row's bits; `cut` truncates the lists (user u keeps (u * cut) % 60 neighbours) so that many users are padded and
    some have none."""
    d = _dict(name)
    if cut:
        d = {u: [v[0][:(u * cut) % 60], v[1][:(u * cut) % 60]] for u, v in d.items()}
    table = graph.UserGraphTable(d, D.K)
    if cut:
        assert (table.n == 0).any() and ((table.n > 0) & (table.n < D.K)).sum() > 10
    for seed in (0, 11):
        np.random.seed(seed)
        a = table.sample(np.random)
        after_a = np.random.randint(0, 2 ** 31, 4)
        np.random.seed(seed)
        b = D.topk_sample_loop(d, D.K)
        after_b = np.random.randint(0, 2 ** 31, 4)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(after_a, after_b)
    empty = table.n == 0
    assert not a[0][empty].any() and not a[1][empty].any()


def _pyg_gcn_norm(edge_index, n):
    """`remove_self_loops`, then `Base_gcn.message` with aggr 'add' (dualgnn.py:327-341)."""
    edge_index = edge_index[:, edge_index[0] != edge_index[1]]
    row, col = edge_index
    deg = torch.zeros(n, dtype=torch.float32).index_add_(0, row, torch.ones(row.numel(), dtype=torch.float32))
    deg_inv_sqrt = deg.pow(-0.5)
    return row, col, deg_inv_sqrt[row] * deg_inv_sqrt[col]


def test_add_values_equal_the_pyg_expression(golden):
    gold = golden("dualgnn_tiny.npz")
    u, i = int(gold["n_users"]), int(gold["n_items"])
    e = torch.stack([torch.from_numpy(gold["inter_row"]), torch.from_numpy(gold["inter_col"]) + u])
    e = torch.cat((e, e[[1, 0]]), dim=1)
    e = torch.cat((e, e[:, :5], torch.tensor([[3, 7], [3, 7]])), dim=1)   # repeated edges and self loops
    row, col, norm = _pyg_gcn_norm(e, u + i)
    dst, src, val = graph.gcn_add_entries(e, u + i)
    assert torch.equal(dst, col) and torch.equal(src, row)
    assert torch.equal(val, norm)                                      # as fp32 bits
    assert val.dtype == torch.float32 and torch.isfinite(val).all()


@pytest.mark.parametrize("mode", ["max", "sum", "", None])
def test_unsupported_aggr_mode_is_refused(mode, tmp_path):
    from mmrec_b200._lib import MMRecError
    from mmrec_b200.models.dualgnn import DualGNN

    class _DS:
        def get_user_num(self):
            return 3

        def get_item_num(self):
            return 2

    class _Loader:
        dataset = _DS()

    cfg = {"USER_ID_FIELD": "u", "ITEM_ID_FIELD": "i", "NEG_PREFIX": "neg_", "train_batch_size": 4, "device": "cpu",
           "end2end": True, "is_multimodal_model": True, "embedding_size": 64, "aggr_mode": mode, "reg_weight": 0.1}
    with pytest.raises(MMRecError, match="aggr_mode"):
        DualGNN(cfg, _Loader())
