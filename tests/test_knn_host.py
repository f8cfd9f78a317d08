"""K7 host side without a GPU: argument errors of the kNN entry points, and `graph._knn`'s dispatch between the two routes
(with CPU stand-ins for the kernels)."""
import torch

from mmrec_b200 import graph


def test_knn_argument_errors_without_a_gpu():
    from mmrec_b200 import _lib
    lib = _lib.load()
    assert lib.mmrec_debug_knn_fallback_rows() == -1                                    # no call yet in this process
    assert lib.mmrec_knn_topk_f32(10, None, 64, 64, 10, None, 11, None, None, None, 0, None) == -1   # k > n
    assert b"knn_topk" in lib.mmrec_last_error()
    assert lib.mmrec_knn_topk_f32(2000, None, 64, 64, 2000, None, 1025, None, None, None, 0, None) == -1   # k > 1024
    assert lib.mmrec_knn_topk_f32(10, None, 64, 64, 10, None, 0, None, None, None, 0, None) == -1     # k < 1
    assert lib.mmrec_knn_topk_f32(10, None, 64, 64, 5, None, 3, None, None, None, 0, None) == -1      # rows NULL, m != n
    assert lib.mmrec_knn_topk_f32(10, None, 64, 64, 10, None, 3, None, None, None, 0, None) == -1     # null pointers
    assert lib.mmrec_knn_topk_f32(10, None, 64, 0, 10, None, 3, None, None, None, 0, None) == -1      # F < 1
    assert lib.mmrec_knn_topk_f32(10, None, 64, 64, 0, 16, 3, None, None, None, 0, None) == 0         # m == 0: nothing to do
    assert lib.mmrec_knn_topk_workspace_bytes(10, 64, 10, 11) == 0
    assert lib.mmrec_knn_topk_workspace_bytes(10, 64, 10, 0) == 0
    assert lib.mmrec_knn_topk_workspace_bytes(7000, 4096, 7000, 10) >= 7000 * 4096 * 2


class _Calls:
    def __init__(self, monkeypatch):
        self.log = []

        def score(u, i, users=None):
            self.log.append(("score", u.shape[1]))
            return u @ i.T

        def mask_topk(s, mask, k, item_offset=0):
            self.log.append(("mask_topk", k))
            return torch.topk(s, k, dim=-1)

        def knn_topk(x, k, rows=None):
            self.log.append(("knn_topk", x.shape[1]))
            q = x if rows is None else x[rows]
            return torch.topk(q @ x.T, k, dim=-1)
        monkeypatch.setattr(graph.ops, "score", score)
        monkeypatch.setattr(graph.ops, "mask_topk", mask_topk)
        monkeypatch.setattr(graph.ops, "knn_topk", knn_topk)


def test_knn_dispatch_by_feature_width(monkeypatch):
    calls = _Calls(monkeypatch)
    g = torch.Generator().manual_seed(0)
    graph._knn(torch.randn(300, 128, generator=g), 5)
    assert {c[0] for c in calls.log} == {"score", "mask_topk"}
    calls.log.clear()
    x = torch.randn(300, 129, generator=g)
    v, i = graph._knn(x, 5)
    assert [c[0] for c in calls.log] == ["knn_topk"]
    assert v.shape == (300, 5) and i.shape == (300, 5)


def test_freedom_rows_are_the_rows_of_the_whole_graph(monkeypatch):
    _Calls(monkeypatch)
    g = torch.Generator().manual_seed(1)
    for F in (64, 256):                                               # both routes
        v, t = torch.randn(200, F, generator=g), torch.randn(200, 96, generator=g)
        pos, col, val, n = graph.freedom_mm_entries(v, t, 7, 0.3)
        rows = torch.tensor([5, 199, 0, 42, 42])
        p2, c2, v2, n2 = graph.freedom_mm_entries(v, t, 7, 0.3, rows=rows)
        assert n2 == n == 200
        for j, r in enumerate(rows.tolist()):
            want = (pos == r)
            got = (p2 == j)
            assert torch.equal(col[want], c2[got])
            assert torch.equal(val[want].view(torch.int32), v2[got].view(torch.int32))
