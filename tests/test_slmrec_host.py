"""SLMRec's host side without a GPU: the adjacency builder `graph.slmrec_adj_entries` for every `adj_type` against a scipy
restatement of `create_adj_mat` (`src/models/slmrec.py:434-479`) and against the reference's own `pre` matrix
(tests/golden/slmrec_tiny.npz), the symmetry flag of `graph.build_slmrec_adj`, and the configurations the class refuses."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

from mmrec_b200 import graph

HERE = os.path.dirname(os.path.abspath(__file__))
ADJ_TYPES = ("plain", "norm", "gcmc", "pre", "mean")


def scipy_adj(row, col, n_users, n_items, adj_type):
    """`create_adj_mat` in scipy with the reference's dtypes, as sorted COO (row, col, fp32 value)."""
    inter = sp.coo_matrix((np.ones(len(row)), (row, col)), shape=(n_users, n_items)).tocsr().astype(np.float32)
    u, i = inter.nonzero()
    n = n_users + n_items
    tmp = sp.csr_matrix((np.ones_like(u, dtype=np.float32), (u, i + n_users)), shape=(n, n))
    adj = tmp + tmp.T

    def single(m):
        rowsum = np.array(m.sum(1))
        with np.errstate(divide="ignore"):
            d_inv = np.power(rowsum, -1).flatten()
        d_inv[np.isinf(d_inv)] = 0.
        return sp.diags(d_inv).dot(m).tocoo()

    if adj_type == "plain":
        out = adj
    elif adj_type == "norm":
        out = single(adj + sp.eye(n))
    elif adj_type == "gcmc":
        out = single(adj)
    elif adj_type == "pre":
        d_inv = np.power(np.array(adj.sum(1)) + 1e-08, -0.5).flatten()
        d_inv[np.isinf(d_inv)] = 0.
        out = sp.diags(d_inv).dot(adj).dot(sp.diags(d_inv))
    else:
        out = single(adj) + sp.eye(n)
    coo = out.tocoo()
    r, c, v = coo.row.astype(np.int64), coo.col.astype(np.int64), coo.data.astype(np.float32)   # torch.FloatTensor(coo.data)
    o = np.lexsort((c, r))
    return r[o], c[o], v[o]


def tiny():
    g = np.load(os.path.join(HERE, "golden", "slmrec_tiny.npz"), allow_pickle=True)
    return g["inter_row"], g["inter_col"], int(g["n_users"]), int(g["n_items"])


def with_isolated_nodes():
    """Users 0, 5, 19 and items 0, 7, 14 have no interaction; one pair is listed twice."""
    rng = np.random.default_rng(3)
    u = rng.choice([1, 2, 3, 4, 6, 8, 11, 12, 17, 18], 60)
    i = rng.choice([1, 2, 3, 5, 6, 9, 10, 13], 60)
    return np.append(u, u[0]), np.append(i, i[0]), 20, 15


@pytest.mark.parametrize("adj_type", ADJ_TYPES)
@pytest.mark.parametrize("graph_fn", [tiny, with_isolated_nodes])
def test_adjacency_equals_the_scipy_restatement(graph_fn, adj_type):
    row, col, nu, ni = graph_fn()
    want = scipy_adj(row, col, nu, ni, adj_type)
    got = graph.slmrec_adj_entries(row, col, nu, ni, adj_type)
    assert got[2].dtype == np.float32
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))


def test_pre_equals_the_reference_matrix():
    g = np.load(os.path.join(HERE, "golden", "slmrec_tiny.npz"), allow_pickle=True)
    assert str(g["cfg_adj_type"]) == "pre"
    idx, val = g["adj_indices"], g["adj_values"]
    o = np.lexsort((idx[1], idx[0]))
    r, c, v = graph.slmrec_adj_entries(g["inter_row"], g["inter_col"], int(g["n_users"]), int(g["n_items"]), "pre")
    assert np.array_equal(r, idx[0][o]) and np.array_equal(c, idx[1][o])
    assert np.array_equal(v.view(np.uint32), val[o].view(np.uint32))


@pytest.mark.parametrize("adj_type", ADJ_TYPES)
def test_symmetric_flag(monkeypatch, adj_type):
    seen = {}

    class Rec:
        @staticmethod
        def from_coo(row, col, val, n_rows, n_cols, sum_duplicates=True, symmetric=False):
            seen.update(symmetric=symmetric, row=row.numpy(), col=col.numpy(), val=val.numpy())
            return "csr"
    monkeypatch.setattr(graph, "CSR", Rec)
    row, col, nu, ni = with_isolated_nodes()
    assert graph.build_slmrec_adj((row, col), nu, ni, "cpu", adj_type) == "csr"
    assert seen["symmetric"] == (adj_type in ("plain", "pre"))
    key = seen["row"] * (nu + ni) + seen["col"]
    tkey = seen["col"] * (nu + ni) + seen["row"]
    o, ot = np.argsort(key), np.argsort(tkey)
    symmetric_bits = np.array_equal(key[o], tkey[ot]) and np.array_equal(seen["val"][o], seen["val"][ot])
    assert symmetric_bits == seen["symmetric"]


class _Data:
    class dataset:
        get_user_num = staticmethod(lambda: 4)
        get_item_num = staticmethod(lambda: 3)


def _config(tmp, **over):
    cfg = {"USER_ID_FIELD": "userID", "ITEM_ID_FIELD": "itemID", "NEG_PREFIX": "neg_", "train_batch_size": 8, "device": "cpu",
           "end2end": False, "is_multimodal_model": True, "data_path": str(tmp) + "/", "dataset": "toy",
           "vision_feature_file": "image_feat.npy", "text_feature_file": "text_feat.npy",
           "ssl_task": "FAC", "mm_fusion_mode": "concat", "init": "xavier"}
    cfg.update(over)
    return cfg


@pytest.mark.parametrize("over,files,why", [
    ({"ssl_task": "FD"}, ("image", "text"), "ssl_task"),
    ({"ssl_task": "FM"}, ("image", "text"), "ssl_task"),
    ({"ssl_task": "FD+FM"}, ("image", "text"), "ssl_task"),
    ({"mm_fusion_mode": "mean"}, ("image", "text"), "mm_fusion_mode"),
    ({"init": "normal"}, ("image", "text"), "embedding_item_ID"),
    ({}, ("image",), "text missing"),
    ({}, ("text",), "image missing"),
    ({"dataset": "kwai"}, ("image", "text"), "kwai"),
])
def test_unsupported_configurations_raise(tmp_path, over, files, why):
    from mmrec_b200._lib import MMRecError
    from mmrec_b200.models.slmrec import SLMRec
    cfg = _config(tmp_path, **over)
    root = tmp_path / cfg["dataset"]
    root.mkdir()
    for f in files:
        np.save(root / f"{f}_feat.npy", np.ones((3, 8), dtype=np.float32))
    with pytest.raises(MMRecError, match=why):
        SLMRec(cfg, _Data())
