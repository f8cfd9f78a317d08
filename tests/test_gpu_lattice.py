"""LATTICE on the GPU: the new values-gradient kernels (`ops.sddmm`, `ops.csr_sym_norm`, `ops.spmm_values`) against torch
and float64, the whole learned graph's gradients against the reference's dense expressions on the device (tiny and baby
shapes), the model class against the golden files recorded from the reference (tests/golden/make_golden_lattice.py), two
epochs through FusedAdam, and the peak memory of a graph-building step at clothing's shape."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import golden_io as G  # noqa: E402
from make_golden_lattice import CASES  # noqa: E402
from test_gpu_models import build  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _pattern(n_rows, n_cols, seed, empty_every=7, hub=None):
    """A power-law CSR pattern (row lengths ~ zipf), every `empty_every`-th row empty, row `hub` with 3000 entries."""
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.zipf(1.6, n_rows), n_cols)
    lens[::empty_every] = 0
    if hub is not None:
        lens[hub] = min(3000, n_cols)
    rows = np.repeat(np.arange(n_rows), lens)
    cols = np.concatenate([rng.choice(n_cols, size=m, replace=False) for m in lens if m] or [np.zeros(0, np.int64)])
    return rows.astype(np.int64), cols.astype(np.int64)


def _csr(dev, rows, cols, n_rows, n_cols, vals=None):
    from mmrec_b200.ops import CSR
    v = None if vals is None else torch.as_tensor(vals, dtype=torch.float32, device=dev)
    return CSR.from_coo(torch.from_numpy(rows).to(dev), torch.from_numpy(cols).to(dev), v, n_rows, n_cols, sum_duplicates=False)


# ------------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 32, 64, 100, 128])
def test_sddmm_matches_the_gathered_dot_product_and_repeats_its_bits(dev, d):
    from mmrec_b200 import ops
    n_rows, n_cols = 5000, 3000
    rows, cols = _pattern(n_rows, n_cols, seed=d, hub=11)
    A = _csr(dev, rows, cols, n_rows, n_cols)
    assert A.nnz == rows.size and int((A.rowptr[1:] == A.rowptr[:-1]).sum()) > 0          # empty rows present
    g = torch.Generator(device="cpu").manual_seed(d)
    P = torch.randn(n_rows, d, generator=g).to(dev)
    Q = torch.randn(n_cols, d, generator=g).to(dev)
    P[3] = float("nan")                                                                    # a NaN row
    out = ops.sddmm_raw(A, P, Q)
    r, c, _ = A.coo()
    want = (P.double()[r] * Q.double()[c]).sum(1)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(out), nan) and bool(nan.any()) == bool((r == 3).any())
    scale = (P.double()[r].abs() * Q.double()[c].abs()).sum(1)
    assert ((out.double() - want).abs()[~nan] <= 4 * d * 2 ** -24 * scale[~nan] + 1e-30).all()
    assert torch.equal(ops.sddmm_raw(A, P, Q).view(torch.int32), out.view(torch.int32))


def test_sddmm_and_spmm_values_refuse_bad_shapes_before_any_launch(dev):
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    rows, cols = _pattern(50, 40, seed=0)
    A = _csr(dev, rows, cols, 50, 40)
    with pytest.raises(MMRecError):
        ops.sddmm_raw(A, torch.zeros(50, 8, device=dev), torch.zeros(41, 8, device=dev))
    with pytest.raises(MMRecError):
        ops.sddmm_raw(A, torch.zeros(50, 8, device=dev), torch.zeros(40, 4, device=dev))
    with pytest.raises(MMRecError):
        ops.spmm_values(A, torch.zeros(A.nnz + 1, device=dev), torch.zeros(40, 8, device=dev))
    with pytest.raises(MMRecError):
        ops.csr_sym_norm(A, torch.zeros(A.nnz, device=dev))                               # not square


def _torch_sym_norm(r, c, a, n):
    rowsum = torch.zeros(n, dtype=a.dtype, device=a.device).index_add(0, r, a)
    d = torch.pow(rowsum, -0.5)
    d = d.masked_fill(torch.isinf(d), 0.0)
    return (d[r] * a) * d[c]


def test_sym_norm_forward_backward_against_torch_autograd_and_float64(dev):
    from mmrec_b200 import ops
    n = 2000
    rows, cols = _pattern(n, n, seed=5, empty_every=9, hub=4)
    # union duplicates: the same (row, col) twice in the COO, summed by the CSR build as the dense sum adds them
    rows = np.concatenate([rows, rows[:500]]); cols = np.concatenate([cols, cols[:500]])
    from mmrec_b200.ops import CSR
    A = CSR.from_coo(torch.from_numpy(rows).to(dev), torch.from_numpy(cols).to(dev), None, n, n, sum_duplicates=True)
    r, c, _ = A.coo()
    g = torch.Generator(device="cpu").manual_seed(0)
    a = torch.rand(A.nnz, generator=g).to(dev)
    neg = 10
    seg = slice(int(A.rowptr[neg]), int(A.rowptr[neg + 1]))
    assert seg.stop > seg.start
    a[seg] = -a[seg].abs()                                                                 # a negative row sum: NaN
    a = a.requires_grad_()
    L = ops.csr_sym_norm(A, a)
    up = torch.randn(A.nnz, generator=g).to(dev)
    (L * up).sum().backward()
    a32 = a.detach().clone().requires_grad_()
    L32 = _torch_sym_norm(r, c, a32, n)
    (L32 * up).sum().backward()
    a64 = a.detach().double().requires_grad_()
    L64 = _torch_sym_norm(r, c, a64, n)
    (L64 * up.double()).sum().backward()
    for got, want in ((L.detach(), L32.detach()), (a.grad, a32.grad)):
        assert torch.equal(torch.isnan(got), torch.isnan(want))
    ok = ~torch.isnan(L64.detach())
    assert bool((~ok).any()) and bool(ok.any())
    assert (L.detach().double() - L64.detach())[ok].abs().max().item() <= 1e-6 * L64.detach()[ok].abs().max().item()
    okg = ~torch.isnan(a64.grad)
    assert (a.grad.double() - a64.grad)[okg].abs().max().item() <= 1e-5 * a64.grad[okg].abs().max().item()
    a2 = a.detach().clone().requires_grad_()
    (ops.csr_sym_norm(A, a2) * up).sum().backward()                                        # the same bits on a second run
    assert torch.equal(a2.grad.view(torch.int32), a.grad.view(torch.int32))


def test_sym_norm_of_an_empty_row_sum_takes_torchs_gradient(dev):
    """A row whose entries sum to exactly 0: d = 0 (inf -> 0) and torch's gradient, NaN through 0 * rowsum^-1.5."""
    from mmrec_b200 import ops
    rows = np.array([0, 0, 1, 1, 2], dtype=np.int64)
    cols = np.array([0, 1, 0, 1, 2], dtype=np.int64)
    A = _csr(dev, rows, cols, 3, 3)
    a = torch.tensor([0.5, -0.5, 1.0, 2.0, 3.0], device=dev, requires_grad=True)
    L = ops.csr_sym_norm(A, a)
    L.sum().backward()
    r, c, _ = A.coo()
    b = a.detach().clone().requires_grad_()
    Lt = _torch_sym_norm(r, c, b, 3)
    Lt.sum().backward()
    assert torch.allclose(L.detach(), Lt.detach(), rtol=1e-6, equal_nan=True)
    assert torch.allclose(a.grad, b.grad, rtol=1e-5, equal_nan=True)


def test_spmm_values_against_torch_sparse_autograd(dev):
    from mmrec_b200 import ops
    n_rows, n_cols, d = 4000, 3000, 64
    rows, cols = _pattern(n_rows, n_cols, seed=9, hub=1)
    A = _csr(dev, rows, cols, n_rows, n_cols)
    r, c, _ = A.coo()
    g = torch.Generator(device="cpu").manual_seed(1)
    v = torch.randn(A.nnz, generator=g).to(dev).requires_grad_()
    X = torch.randn(n_cols, d, generator=g).to(dev).requires_grad_()
    up = torch.randn(n_rows, d, generator=g).to(dev)
    Y = ops.spmm_values(A, v, X)
    (Y * up).sum().backward()
    v2, X2 = v.detach().double().requires_grad_(), X.detach().double().requires_grad_()
    S = torch.sparse_coo_tensor(torch.stack([r, c]), v2, (n_rows, n_cols))
    Y2 = torch.sparse.mm(S, X2)
    (Y2 * up.double()).sum().backward()
    for got, want in ((Y.detach(), Y2.detach()), (v.grad, v2.grad), (X.grad, X2.grad)):
        assert (got.double() - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    v3, X3 = v.detach().clone().requires_grad_(), X.detach().clone().requires_grad_()
    (ops.spmm_values(A, v3, X3) * up).sum().backward()
    assert torch.equal(v3.grad, v.grad) and torch.equal(X3.grad, X.grad)


# ------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------
def _env(shape, mods, seed=0):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_")
    u, i, e, d, f = synth.SHAPES[shape]
    g = synth.make_graph(u, i, e, seed=seed)
    if shape == "tiny":
        v, t = synth.make_features(i, f, seed=1)
    else:
        rng = np.random.default_rng(1)
        v, t = rng.standard_normal((i, f), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, v if "v" in mods else None, t if "t" in mods else None)
    return os.path.join(tmp, "data") + "/"


@pytest.fixture(scope="module")
def envs(dev):
    return {m: _env("tiny", m) for m in ("vt", "v", "t")}


def _sub(gold, p):
    out = {}
    for k in gold.files:
        if k.startswith(p) and not any(k.startswith(q) for q in CASES if q and q != p and len(q) > len(p)):
            out[k[len(p):]] = gold[k]
    return out


def _overrides(p):
    return dict(CASES[p][0])


def _dense(gold, key, n):
    out = torch.zeros(n, n, dtype=torch.float64)
    out[tuple(torch.from_numpy(gold[key + ".index"]).long())] = torch.from_numpy(gold[key + ".values"]).double()
    return out


def _csr_dense(A):
    r, c, v = A.coo()
    return torch.zeros(A.n_rows, A.n_cols, dtype=torch.float64).index_put_((r.cpu(), c.cpu()), v.detach().cpu().double(),
                                                                           accumulate=True)


def _close_graph(got, want, tol):
    assert torch.equal(got != 0, want != 0), "the pattern differs"
    assert (got - want).abs().max().item() <= tol * want.abs().max().item()


def _check_grads(gold, model, tag, tol):
    named = dict(model.named_parameters())
    rec = [k[len(tag + "grad."):] for k in G.recorded(gold, tag + "grad.")]
    if tag == "plain." and not rec:                                    # recorded for the first case only
        return
    assert set(rec) == {k for k, q in named.items() if q.grad is not None}
    for k in rec:
        assert G.rel(gold, tag + "grad." + k, named[k].grad.cpu().numpy()) < tol, f"{tag}grad {k}"


@pytest.mark.parametrize("p", list(CASES))
def test_lattice_matches_reference(envs, golden, p):
    from mmrec_b200.common.trainer import Trainer
    full = golden("lattice_tiny.npz")
    gold = _sub(full, p)
    config, train, valid, test, model = build("LATTICE", envs[CASES[p][1]], _overrides(p))
    dev = config["device"]
    n = model.n_items
    graph_key = p + "item_adj" if p + "item_adj.index" in full.files else "item_adj"   # recorded where it differs from the first case's
    init = {k[len("init_sha256."):]: str(v) for k, v in gold.items() if k.startswith("init_sha256.")}
    assert G.init_digests(model) == init, "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    r, c, v = model.norm_adj.coo()
    assert np.array_equal(np.stack([r.cpu().numpy(), c.cpu().numpy()]), full["norm_adj_indices"])
    assert np.array_equal(v.cpu().numpy(), full["norm_adj_values"])
    for name, m in (("image_original_adj", "v"), ("text_original_adj", "t")):
        if m in CASES[p][1]:
            _close_graph(_csr_dense(getattr(model, name)), _dense(full, name, n), 1e-6)
    model.train()
    model.pre_epoch_processing()
    for tag in ("build.", "plain."):
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(torch.from_numpy(gold[tag + "batch"]).to(dev))
        if tag == "build.":
            _close_graph(_csr_dense(model.item_adj), _dense(full, graph_key, n), 1e-5)
            if not p:                                                     # forward's embeddings: recorded for the first case
                u_g, i_g = model.forward(model.norm_adj)
                assert G.rel(gold, "build.u_g", u_g.detach().cpu().numpy()) < 1e-5
                assert G.rel(gold, "build.i_g", i_g.detach().cpu().numpy()) < 1e-5
        loss.backward()
        np.testing.assert_allclose(loss.item(), gold[tag + "loss"][0], rtol=1e-5)
        _check_grads(gold, model, tag, 1e-4)
    for name in ("image_trs", "text_trs"):                              # not read on an ordinary batch
        if hasattr(model, name):
            assert getattr(model, name).weight.grad is None
    model.zero_grad(set_to_none=True)
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
        _close_graph(_csr_dense(model.item_adj), _dense(full, graph_key, n), 1e-5)   # the same graph, built again
        adj = model.item_adj
        idx = model.full_sort_topk(eb, 50).cpu()
        assert model.item_adj is adj                                     # built once per evaluation
        want = torch.from_numpy(gold["topk50"]).long()
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10
        m = m.cpu().double()
        scale = m[m > -1e9].abs().max().item()
        diff = idx != want
        gap = (m.gather(1, idx) - m.gather(1, want)).abs()
        assert (gap[diff] <= 1e-5 * scale).all() and diff.float().mean().item() < 0.05
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_lattice_trajectory_through_fused_adam(envs, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches: per-batch losses, per-epoch metrics and the final
    weights; `image_trs` / `text_trs` get a gradient on the graph-building batch only, and FusedAdam leaves them alone on
    the others."""
    gold = golden("traj_lattice_tiny.npz")
    config, train, valid, test, model = build("LATTICE", envs["vt"], {})
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches = gold["batches"]
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    b = 0
    for ep, nb in enumerate(gold["batches_per_epoch"]):
        model.pre_epoch_processing()
        model.train()
        for j in range(int(nb)):
            trainer.optimizer.zero_grad()
            loss = model.calculate_loss(torch.from_numpy(batches[:, offs[b]:offs[b + 1]].copy()).to(dev))
            np.testing.assert_allclose(loss.item(), gold["losses"][b], rtol=1e-5)
            loss.backward()
            w = model.image_trs.weight.detach().clone()
            assert (model.image_trs.weight.grad is not None) == (j == 0)
            trainer.optimizer.step()
            assert torch.equal(model.image_trs.weight.detach(), w) == (j > 0)
            b += 1
        trainer.lr_scheduler.step()
        v = trainer.evaluate(valid)
        t = trainer.evaluate(test, is_test=True)
        np.testing.assert_allclose([v[k] for k in names], gold["valid"][ep], atol=2e-4)
        np.testing.assert_allclose([t[k] for k in names], gold["test"][ep], atol=2e-4)
    assert b == int(gold["n_steps"])
    for k, q in model.state_dict().items():
        want = gold["final." + k]
        assert np.linalg.norm(q.cpu().numpy() - want) <= 1e-4 * max(np.linalg.norm(want), 1e-30), k


def _dense_item_adj(model):
    """The reference's dense expressions (`lattice.py:132-157`, `utils.py:119-137`) on the device, from the model's own
    parameters: image_feats, build_sim, build_knn_neighbourhood, the weighted sums and compute_normalized_laplacian."""
    def build_sim(x):
        xn = x.div(torch.norm(x, p=2, dim=-1, keepdim=True))
        return torch.mm(xn, xn.transpose(1, 0))

    def knn(adj, k):
        val, ind = torch.topk(adj, k, dim=-1)
        return torch.zeros_like(adj).scatter_(-1, ind, val)

    def lap(adj):
        d = torch.pow(torch.sum(adj, -1), -0.5)
        d[torch.isinf(d)] = 0.
        dm = torch.diagflat(d)
        return torch.mm(torch.mm(dm, adj), dm)

    w = torch.softmax(model.modal_weight, dim=0)
    img = knn(build_sim(model.image_trs(model.image_embedding.weight)), model.knn_k)
    txt = knn(build_sim(model.text_trs(model.text_embedding.weight)), model.knn_k)
    orig = w[0] * model.image_original_adj.to_dense() + w[1] * model.text_original_adj.to_dense()
    return (1 - model.lambda_coeff) * lap(w[0] * img + w[1] * txt) + model.lambda_coeff * orig


@pytest.mark.parametrize("shape", ["tiny", "baby"])
def test_learned_graph_gradients_against_the_dense_reference_on_the_device(dev, shape):
    """h = item_adj^2 item_id_embedding through the learned graph, sparse against dense: the graph, h and the gradients of
    modal_weight, both projections, both feature tables and the item table."""
    from mmrec_b200 import ops
    torch.backends.cuda.matmul.allow_tf32 = False
    config, train, valid, test, model = build("LATTICE", _env(shape, "vt"), {"n_layers": 2})
    n = model.n_items
    gen = torch.Generator(device="cpu").manual_seed(3)
    up = torch.randn(n, model.embedding_dim, generator=gen).to(dev)
    with torch.no_grad():
        model.modal_weight.copy_(torch.tensor([0.3, 0.8]))
    params = [model.modal_weight, model.image_trs.weight, model.image_trs.bias, model.text_trs.weight, model.text_trs.bias,
              model.image_embedding.weight, model.text_embedding.weight, model.item_id_embedding.weight]
    adj = model.build_learned_graph()
    h = model.item_id_embedding.weight
    for _ in range(2):
        h = ops.spmm_values(adj, adj.vals, h)
    got = torch.autograd.grad((h * up).sum(), params)
    dense = _dense_item_adj(model)
    hd = torch.mm(dense, torch.mm(dense, model.item_id_embedding.weight))
    want = torch.autograd.grad((hd * up).sum(), params)
    gd = _csr_dense(adj)
    wd = dense.detach().double().cpu()
    mismatch = ((gd != 0) != (wd != 0)).float().sum().item() / max((wd != 0).sum().item(), 1)
    assert mismatch < 1e-3, f"learned pattern differs in {mismatch:.2%} of the entries"
    if mismatch == 0:
        assert (gd - wd).abs().max().item() <= 1e-5 * wd.abs().max().item()
    assert (h - hd).norm().item() <= 1e-4 * hd.norm().item()
    names = ["modal_weight", "image_trs.weight", "image_trs.bias", "text_trs.weight", "text_trs.bias", "image_embedding",
             "text_embedding", "item_id_embedding"]
    for name, a, b in zip(names, got, want):
        assert (a - b).norm().item() <= 1e-3 * b.norm().item(), name
    del dense, hd, want
    torch.cuda.empty_cache()


def test_graph_building_step_at_clothing_shape_allocates_no_item_by_item_matrix(dev):
    """A graph-building `calculate_loss` + backward at clothing's 23 000 items: beside the dense gradients of the two
    feature tables, the peak above the model stays below half of one dense [I, I] fp32 matrix (2.1 GB); the largest
    intermediate is a 256 MiB block of similarities."""
    config, train, valid, test, model = build("LATTICE", _env("clothing", "vt"), {"train_batch_size": 2048})
    n = model.n_items
    batch = next(iter(train)).to(config["device"])
    model.train()
    model.pre_epoch_processing()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss = model.calculate_loss(batch)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    dense = 4 * n * n
    tables = 4 * (model.image_embedding.weight.numel() + model.text_embedding.weight.numel())   # their dense gradients
    assert peak - tables < 0.5 * dense, \
        f"peak {peak / 2**20:.0f} MiB above the model ({tables / 2**20:.0f} MiB table gradients), one [I, I] matrix is {dense / 2**20:.0f} MiB"
