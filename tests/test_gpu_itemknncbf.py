"""ItemKNNCBF on the device.  K7's shrink route (`ops.knn_topk(.., norms=, shrink=)`) against the exact route bit for bit;
K9 (csrc/sparse_score.cu): `ops.sparse_scores` against the ordered sum of tests/itemknncbf_oracle.py and
`ops.sparse_score_topk` against `sparse_scores` + `mask_topk` bit for bit; the model class on `tiny` against the reference's
golden file, and its memory at clothing's shape."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import itemknncbf_oracle as KO  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- K7, shrink route -----------------------------------------------------------------------------------------------
def _exact_shrink(x, k, shrink, rows=None, norms=None):
    """The exact route: CUDA-core score chain, the elementwise denominator (torch: multiply, add, divide), mask_topk."""
    from mmrec_b200 import ops
    n = x.shape[0]
    norms = torch.norm(x, p=2, dim=-1) if norms is None else norms
    rows = torch.arange(n, device=x.device) if rows is None else rows
    vals, idxs = [], []
    ops.set_score_path("simt")
    try:
        for r0 in range(0, rows.numel(), 2048):
            rr = rows[r0:r0 + 2048]
            s = ops.score(x, x, rr)
            s = s / (norms[rr][:, None] * norms[None, :] + shrink)
            v, i = ops.mask_topk(s, None, k)
            vals.append(v)
            idxs.append(i)
    finally:
        ops.set_score_path("auto")
    return torch.cat(vals), torch.cat(idxs)


def _table(n, F, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, F, generator=g, device="cuda")


@pytest.mark.parametrize("n", [120, 7000, 23000])
@pytest.mark.parametrize("F", [256, 8192])
@pytest.mark.parametrize("shrink", [0.0, 10.0, 1e4])
def test_knn_shrink_equals_exact_route(n, F, shrink):
    from mmrec_b200 import ops
    _dev()
    x = _table(n, F, seed=n + F)
    k = 10
    val, idx = ops.knn_topk(x, k, shrink=shrink)
    fb = ops.knn_fallback_rows()
    ev, ei = _exact_shrink(x, k, shrink)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))
    if n >= 7000:
        assert fb == 0, f"{fb} rows took the exact route"


def test_knn_shrink_rows_subset_and_ties():
    from mmrec_b200 import ops
    _dev()
    x = _table(7000, 512, seed=3)
    x[5] = x[3]                                                       # exact ties
    x[100] = x[3]
    x[7] = 0.0                                                        # a zero row
    rows = torch.randperm(7000, generator=torch.Generator().manual_seed(0))[:700].cuda()
    rows[:3] = torch.tensor([3, 5, 7])
    for shrink in (10.0, 0.0):
        val, idx = ops.knn_topk(x, 20, rows=rows, shrink=shrink)
        ev, ei = _exact_shrink(x, 20, shrink, rows=rows)
        assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev)), shrink
    assert ops.knn_fallback_rows() == 700                             # shrink 0 with a zero norm: 0 / 0, the exact route
    assert torch.isnan(val[2]).any()


def test_knn_shrink_nan_row_takes_the_exact_route():
    from mmrec_b200 import ops
    _dev()
    x = _table(3000, 256, seed=4)
    x[9, 17] = float("nan")
    val, idx = ops.knn_topk(x, 10, shrink=10.0)
    assert ops.knn_fallback_rows() == 3000
    ev, ei = _exact_shrink(x, 10, 10.0)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))


def test_knn_shrink_largest_shape_sampled_rows():
    """125 037 items x 8192 (one GPU's share of configs[4]): a sample of rows against the exact route."""
    from mmrec_b200 import ops
    _dev()
    x = _table(125037, 8192, seed=5)
    rows = torch.randperm(125037, generator=torch.Generator().manual_seed(1))[:256].cuda()
    val, idx = ops.knn_topk(x, 10, rows=rows, shrink=10.0)
    assert ops.knn_fallback_rows() == 0
    ev, ei = _exact_shrink(x, 10, 10.0, rows=rows)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))


# ---- K9 -------------------------------------------------------------------------------------------------------------
def _round20(a):
    """fp32 values with 20 significand bits: products with the R values below stay exact, so fmaf = multiply + add."""
    b = np.asarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFFFF0)
    return b.view(np.float32)


def _graphs(n_users, n_items, knn_k, seed, unit=True, long_user=None):
    """R (CSR [U, I], empty rows included) and S (CSR [I, I], knn_k distinct columns per row), host arrays and device CSRs."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(n_users):
        d = 0 if u % 17 == 0 else int(rng.integers(1, 40))
        if long_user is not None and u == long_user:
            d = 300
        c = rng.choice(n_items, size=d, replace=False)
        rows += [u] * d
        cols += list(c)
    rows, cols = np.array(rows, np.int64), np.array(cols, np.int64)
    rv = np.ones(len(rows), np.float32) if unit else rng.choice(np.array([0.5, 1.0, 2.0, 3.0, 1.5], np.float32), len(rows))
    sv = _round20(rng.standard_normal((n_items, knn_k)).astype(np.float32) + 0.3)
    si = np.stack([rng.choice(n_items, size=knn_k, replace=False) for _ in range(n_items)])
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    R = ops.CSR.from_coo(t(rows), t(cols), t(rv), n_users, n_items)
    S = ops.CSR.from_coo(t(np.repeat(np.arange(n_items), knn_k)), t(si.reshape(-1)), t(sv.reshape(-1)), n_items, n_items)
    return (rows, cols, rv, sv, si), R, S


@pytest.mark.parametrize("unit", [True, False])
def test_sparse_scores_equal_the_ordered_sum(unit):
    from mmrec_b200 import ops
    dev = _dev()
    (rows, cols, rv, sv, si), R, S = _graphs(400, 3000, 10, seed=1, unit=unit)
    users = np.array([0, 5, 5, 17, 399, 34, 5, 1, 200], np.int64)         # empty histories (0, 17, 34), repeated users
    got = ops.sparse_scores(R, S, torch.from_numpy(users).to(dev))
    want = KO.ordered_scores(rows, cols, rv, 400, sv, si, users=users)
    assert torch.equal(_bits(got.cpu()), _bits(torch.from_numpy(want)))
    assert not got[0].any() and not got[3].any()
    full = ops.sparse_scores(R, S)
    assert full.shape == (400, 3000) and torch.equal(_bits(full[users].cpu()), _bits(got.cpu()))


def _mask_for(users, R_rows, R_cols, extra=None):
    m = [(b, c) for b, u in enumerate(users) for c in R_cols[R_rows == u]]
    if extra:
        m += extra
    m = np.array(m, np.int64).reshape(-1, 2).T
    return m


@pytest.mark.parametrize("k", [1, 20, 50, 1024])
@pytest.mark.parametrize("unit", [True, False])
def test_sparse_score_topk_equals_scores_plus_mask_topk(k, unit):
    from mmrec_b200 import ops
    dev = _dev()
    (rows, cols, rv, sv, si), R, S = _graphs(600, 4000, 10, seed=2 + k, unit=unit)
    users = np.concatenate([np.arange(600), [3, 3, 17]]).astype(np.int64)
    # masks over candidates and non-candidates, duplicates, an item outside the catalogue
    mask = _mask_for(users, rows, cols, extra=[(1, 5), (1, 5), (2, 3999), (4, 4000)])
    tu, tm = torch.from_numpy(users).to(dev), torch.from_numpy(mask).to(dev)
    val, idx = ops.sparse_score_topk(R, S, tu, tm, k)
    assert ops.sparse_topk_fallback_rows() == 0
    ev, ei = ops.mask_topk(ops.sparse_scores(R, S, tu), tm, k)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))


@pytest.mark.parametrize("route", ["sorted", "unsorted", "large"])
def test_sparse_score_topk_mask_routes_and_wrapping_columns(route):
    """Each route of the batch mask CSR (rows in order, out of order, B > 8192), with a column 2^32 + j per row, j the
    row's unmasked top-1: mmrec_mask_f32 ignores such a column although its low 32 bits name item j, and so must K9."""
    from mmrec_b200 import ops
    dev = _dev()
    (rows, cols, rv, sv, si), R, S = _graphs(600, 4000, 10, seed=7)
    users = np.arange(9000 if route == "large" else 600, dtype=np.int64) % 600
    tu, tm = torch.from_numpy(users).to(dev), torch.from_numpy(_mask_for(users, rows, cols)).to(dev)
    sc = ops.sparse_scores(R, S, tu)
    _, top = ops.mask_topk(sc.clone(), tm, 1)
    m = torch.cat([tm, torch.stack([torch.arange(len(users), device=dev), top[:, 0] + 2 ** 32])], 1)
    order = torch.randperm(m.shape[1]) if route == "unsorted" else torch.argsort(m[0].cpu(), stable=True)
    m = m[:, order.to(dev)]
    val, idx = ops.sparse_score_topk(R, S, tu, m, 20)
    assert ops.sparse_topk_fallback_rows() == 0
    ev, ei = ops.mask_topk(sc.clone(), m, 20)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))


def test_sparse_score_topk_ranking_cases():
    """Few candidates (the +0.0 class fills the rest, masked items skipped), negative sums, a -0.0 sum, k beyond the
    unmasked items (the -1e10 entries follow), and a history whose products overflow shared memory (the unfused route)."""
    from mmrec_b200 import ops
    dev = _dev()
    n_items = 64
    # S: item i -> columns (i + 1 .. i + 3) % n with values +1, -2, tiny negative
    si = np.stack([(np.arange(3) + i + 1) % n_items for i in range(n_items)])
    sv = np.tile(np.array([1.0, -2.0, -2.0 ** -60], np.float32), (n_items, 1))
    sv[10] = [-1.0, -0.5, -2.0 ** -60]
    R_rows = np.array([0, 1, 1, 2, 3, 3, 3], np.int64)
    R_cols = np.array([10, 20, 40, 30, 0, 1, 2], np.int64)
    rv = np.array([1.0, 1.0, 1.0, 2.0 ** -100, 1.0, 1.0, 1.0], np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    R = ops.CSR.from_coo(t(R_rows), t(R_cols), t(rv), 4, n_items)
    S = ops.CSR.from_coo(t(np.repeat(np.arange(n_items), 3)), t(si.reshape(-1)), t(sv.reshape(-1)), n_items, n_items)
    users = t(np.array([0, 1, 2, 3, 3], np.int64))
    sc = ops.sparse_scores(R, S, users)
    assert float(sc[2, 33]) == 0.0 and torch.signbit(sc[2, 33])    # a sum whose only product underflows: -0.0
    # batch row 4 masks all but 5 items: k = 50 runs into the -1e10 entries
    mask = [(0, 11), (0, 50), (1, 21), (1, 0), (3, 2)] + [(4, c) for c in range(5, n_items)]
    tm = t(np.array(mask, np.int64).T)
    for k in (1, 5, 20, 50, 64):
        val, idx = ops.sparse_score_topk(R, S, users, tm, k)
        assert ops.sparse_topk_fallback_rows() == 0
        ev, ei = ops.mask_topk(sc.clone(), tm, k)
        assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev)), k
        for b in range(5):
            rv_, ri_ = KO.dense_rank(sc[b].cpu().numpy(), [c for r, c in mask if r == b], k)
            assert np.array_equal(ri_, idx[b].cpu().numpy()), (k, b)
    # overflow: one history of 300 items x 10 neighbours > 2048 products
    (rows, cols, rv2, sv2, si2), R2, S2 = _graphs(50, 3000, 10, seed=9, long_user=7)
    users = t(np.arange(50, dtype=np.int64))
    tm = t(_mask_for(np.arange(50), rows, cols))
    val, idx = ops.sparse_score_topk(R2, S2, users, tm, 50)
    assert ops.sparse_topk_fallback_rows() == 1
    ev, ei = ops.mask_topk(ops.sparse_scores(R2, S2, users), tm, 50)
    assert torch.equal(idx, ei) and torch.equal(_bits(val), _bits(ev))


# ---- the model -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import tempfile
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_")
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, v, t)
    return os.path.join(tmp, "data") + "/"


@pytest.mark.parametrize("prefix,shrink", [("s10_", 10), ("s0_", 0)])
def test_itemknncbf_matches_reference(env, prefix, shrink):
    from test_gpu_models import build
    from mmrec_b200.common.trainer import Trainer
    gold = np.load(os.path.join(HERE, "golden", "itemknncbf_tiny.npz"), allow_pickle=True)
    G = lambda k: gold[prefix + k]
    config, train, valid, test, model = build("ItemKNNCBF", env, {"shrink": [shrink]})
    dev = config["device"]
    assert [k for k, _ in model.named_parameters()] == ["dummy_embeddings"]
    assert np.array_equal(model.dummy_embeddings.detach().cpu().numpy(), G("dummy_embeddings"))
    assert not any(t.numel() >= model.n_items ** 2 for t in list(model.parameters()) + list(model.buffers()))
    # the kNN graph: same neighbours, except near ties the fp64 similarity cannot separate
    feats = KO.features(model.v_feat, model.t_feat).double().cpu()
    nrm = feats.norm(dim=-1, keepdim=True)
    sim64 = (feats @ feats.T) / (nrm * nrm.T + shrink)
    S = model.item_sim
    k = int(G("cfg_knn_k"))
    gi = S.colidx.view(-1, k).cpu().numpy()
    want_i = np.sort(G("knn_ind"), axis=1)
    for r in np.nonzero((gi != want_i).any(axis=1))[0]:
        a, b = set(gi[r]), set(want_i[r])
        gap = abs(float(sim64[r, list(a - b)].min()) - float(sim64[r, list(b - a)].max()))
        assert gap < 1e-6, f"row {r}: kNN differs beyond a near tie ({gap})"
    eb = [torch.from_numpy(G("eval_users")).to(dev), torch.from_numpy(G("eval_mask")).to(dev)]
    scores = model.full_sort_predict(eb)
    want = G("scores")
    assert float(np.abs(scores.cpu().numpy() - want).max()) <= 1e-6 * float(np.abs(want).max())
    names = [str(x) for x in G("metric_names")]
    res = {}
    for fused in (True, False):
        config["use_fused_topk"] = fused
        tr = Trainer(config, model)
        res[fused] = ([tr.evaluate(valid)[k] for k in names], [tr.evaluate(test, is_test=True)[k] for k in names])
    assert res[True] == res[False]
    # The reference ranks with CPU torch.topk, whose order among equal scores is its own.  On `tiny` a user's candidates
    # (deg(u) * knn_k products) often number fewer than 50, so the tail of a top-20 / top-50 is the +0.0 class, where this
    # package takes ascending item index.  So: the reference's own scores_matrix, ranked on the device under that tie rule,
    # must give this model's metrics exactly, and every metric whose cut-off stays above the +0.0 class (@5, @10) must equal
    # the golden file's.
    sm = torch.from_numpy(G("scores_matrix")).to(dev)

    class RefScores(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(2, device=dev))

        def full_sort_predict(self, interaction):
            return sm[interaction[0]].clone()
    config["use_fused_topk"] = False
    tr = Trainer(config, RefScores())
    ref_tie = ([tr.evaluate(valid)[k] for k in names], [tr.evaluate(test, is_test=True)[k] for k in names])
    np.testing.assert_allclose(res[True][0], ref_tie[0], atol=1e-9, rtol=0)
    np.testing.assert_allclose(res[True][1], ref_tie[1], atol=1e-9, rtol=0)
    top = [j for j, nm in enumerate(names) if nm.endswith("@5") or nm.endswith("@10")]
    assert len(top) >= 4
    np.testing.assert_allclose(np.array(res[True][0])[top], G("metric_values")[top], atol=1e-9, rtol=0)
    np.testing.assert_allclose(np.array(res[True][1])[top], G("test_metric_values")[top], atol=1e-9, rtol=0)


def test_itemknncbf_memory_at_clothing_shape(tmp_path):
    """Build at clothing's shape (23 000 items, F = 8192 concatenated) and evaluate every user: the peak above the feature
    tables and the kNN build's fp16 pack stays far below the reference's dense [I, I] + [U, I] (2.1 + 3.7 GB)."""
    from test_gpu_models import build
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.utils import synth
    _dev()
    u, i, e, d, f = synth.SHAPES["clothing"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(str(tmp_path), "tiny", g, v, t)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    config, train, valid, test, model = build("ItemKNNCBF", str(tmp_path) + "/", {"eval_batch_size": 4096})
    Trainer(config, model).evaluate(test, is_test=True)
    peak = torch.cuda.max_memory_allocated() - base
    feats = 2 * i * f * 4                                             # v_feat, t_feat
    pack = 2 * i * 2 * f                                              # cat(v, t) in fp16: the kNN build's operand
    extra = peak - feats - 2 * i * f * 4 - pack                       # also minus the concatenated fp32 copy
    print(f"ItemKNNCBF clothing shape: peak {peak / 2**30:.2f} GiB, above tables + concatenation + pack {extra / 2**30:.3f} GiB")
    assert extra < 0.25 * (2.1 + 3.7) * 2**30
