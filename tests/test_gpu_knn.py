"""K7 (csrc/knn_cf.cu): `ops.knn_topk` against the route it replaces -- `ops.score` (exact CUDA-core kernel at F > 128) then
`ops.mask_topk` -- on the same normalised table.  Values bitwise, indices exactly."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _normalise(x):
    return x.div(torch.norm(x, p=2, dim=-1, keepdim=True)).contiguous()


def _old_route(cn, k, rows=None):
    from mmrec_b200 import ops
    q = cn if rows is None else cn.index_select(0, rows)
    step = max(128, (256 << 20) // (4 * cn.shape[0]))
    vals, inds = [], []
    for s in range(0, q.shape[0], step):
        v, i = ops.mask_topk(ops.score(q[s:s + step], cn), None, k)
        vals.append(v); inds.append(i)
    return torch.cat(vals), torch.cat(inds)


def _assert_same(new, old):
    (vn, i_n), (vo, io) = new, old
    assert vn.shape == vo.shape and i_n.shape == io.shape
    bad = (vn.view(torch.int32) != vo.view(torch.int32)).any(dim=1) | (i_n != io).any(dim=1)
    assert not bool(bad.any()), f"{int(bad.sum())} rows differ, first {int(bad.nonzero()[0])}"


def _table(n, F, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, F, generator=g, device="cuda")


@pytest.mark.parametrize("n,F", [(7000, 4096), (18000, 4096), (23000, 4096), (7000, 384), (7000, 200), (7000, 4100)])
def test_knn_topk_bitwise_equals_score_then_topk(n, F):
    from mmrec_b200 import ops
    _dev()
    cn = _normalise(_table(n, F, n + F))
    for k in (1, 10, 50):
        _assert_same(ops.knn_topk(cn, k), _old_route(cn, k))
    assert ops.knn_fallback_rows() >= 0


def test_knn_topk_one_gpu_share_of_the_large_catalogue_needs_no_fallback():
    from mmrec_b200 import ops
    _dev()
    cn = _normalise(_table(125037, 4096, 7))
    new = ops.knn_topk(cn, 10)
    assert ops.knn_fallback_rows() == 0
    _assert_same(new, _old_route(cn, 10))


def test_knn_topk_ties_and_clusters_take_the_exact_route_and_still_match():
    from mmrec_b200 import ops
    _dev()
    g = torch.Generator(device="cuda").manual_seed(3)
    n, F = 8000, 4096
    x = torch.randn(n, F, generator=g, device="cuda")
    base = torch.randn(1, F, generator=g, device="cuda")
    x[:5000] = base + 1e-4 * torch.randn(5000, F, generator=g, device="cuda")   # one tight cluster: too many candidates
    x[6000:6500] = x[5000:5500]                                                 # exact duplicates: ties at cosine 1
    x[6500:6600] = x[100:200]                                                   # duplicates inside the cluster
    x[7000:7300] = x[5500:5800].flip(0)
    cn = _normalise(x)
    for k in (1, 10, 50):
        new = ops.knn_topk(cn, k)
        assert ops.knn_fallback_rows() > 0
        _assert_same(new, _old_route(cn, k))


def test_knn_topk_query_rows_subset():
    from mmrec_b200 import ops
    _dev()
    cn = _normalise(_table(9000, 4096, 11))
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = torch.randint(0, 9000, (1500,), generator=g, device="cuda")
    for k in (10, 50):
        _assert_same(ops.knn_topk(cn, k, rows), _old_route(cn, k, rows))


def test_knn_topk_non_finite_table_takes_the_existing_route_whole():
    from mmrec_b200 import ops
    _dev()
    x = _table(3000, 4096, 13)
    x[17] = 0.0                                                        # normalises to NaN
    cn = _normalise(x)
    assert bool(torch.isnan(cn).any())
    new = ops.knn_topk(cn, 10)
    assert ops.knn_fallback_rows() == 3000
    _assert_same(new, _old_route(cn, 10))


def _old_dispatch(monkeypatch):
    """graph._knn with ops.knn_topk replaced by the route it replaces."""
    from mmrec_b200 import graph
    monkeypatch.setattr(graph.ops, "knn_topk", lambda cn, k, rows=None: _old_route(cn, k, rows))


def _csr_equal(a, b):
    assert a.n_rows == b.n_rows and a.n_cols == b.n_cols and a.nnz == b.nnz
    assert torch.equal(a.rowptr, b.rowptr)
    assert torch.equal(a.colidx[:a.nnz], b.colidx[:b.nnz])
    assert torch.equal(a.vals[:a.nnz].view(torch.int32), b.vals[:b.nnz].view(torch.int32))


def _features():
    return _table(7000, 4096, 21), _table(7000, 384, 22)


def test_freedom_and_mgcn_item_graphs_equal_the_old_route(monkeypatch):
    """The builders FREEDOM (`models/freedom.py`: mm_adj) and MGCN (`models/mgcn.py`: image / text_original_adj) call."""
    from mmrec_b200 import graph
    _dev()
    v, t = _features()
    # MGCN's degree is a float scatter-add (`index_add_`, as the reference's `scatter_add`, utils.py:141): atomics whose
    # order varies between runs unless torch's deterministic mode picks its ordered kernel.  Both builds run under it.
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        new = [graph.build_freedom_mm_adj(v, t, 10, 0.1), graph.build_mgcn_knn_adj(v, 10), graph.build_mgcn_knn_adj(t, 10)]
        _old_dispatch(monkeypatch)
        old = [graph.build_freedom_mm_adj(v, t, 10, 0.1), graph.build_mgcn_knn_adj(v, 10), graph.build_mgcn_knn_adj(t, 10)]
    finally:
        torch.use_deterministic_algorithms(was)
    for a, b in zip(new, old):
        _csr_equal(a, b)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_freedom_mm_rows_equal_the_single_gpu_graph(world):
    from mmrec_b200 import graph
    from mmrec_b200.sharded import ItemShard
    dev = _dev()
    v, t = _features()
    n = v.shape[0]
    full = graph.build_freedom_mm_adj(v, t, 10, 0.1)
    r, c, val = (x.cpu().numpy() for x in full.coo())
    inter_u, inter_i = np.arange(n) % 50, np.arange(n)
    for rank in range(world):
        shard = ItemShard(inter_u, inter_i, 50, n, rank, world)
        _csr_equal(shard.freedom_mm_csr(v, t, 10, 0.1, dev), shard.mm_csr(r, c, val, dev))
