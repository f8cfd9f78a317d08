"""DualGNN on the GPU: the two towers' propagation as one width-128 `ops.propagate_sum`, the user-graph aggregation as
`ops.spmm` on the epoch's user graph, and the model class against the golden files recorded from the reference
(tests/golden/make_golden_dualgnn.py).

- Propagation: x + A x + A (A x) on [x_v | x_t] equals two width-64 propagations and the float64 result within the fp32
  reorder bound, forward and backward, for the 'add' and 'mean' adjacencies; on exactly representable operands it equals
  float64 bit for bit.
- User graph: `spmm(G, X, base=X)` against autograd of the reference's `X + matmul(w.unsqueeze(1), X[idx]).squeeze()`
  on the device; bit for bit on exact operands with repeated neighbours and users without any; and at clothing's 40 000
  users the op's peak allocation, forward and backward, stays below an eighth of the reference's [U, 40, 64] fp32 gather.
- Model: initial state, the float64 scores before any forward, the epoch sample, the mutated batch, the towers, the loss,
  every gradient, the scores and metrics, also text-only; two epochs through FusedAdam; `full_sort_topk` against
  `mask_topk` of `full_sort_predict`."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import dualgnn_golden as D  # noqa: E402
import golden_io as G  # noqa: E402
from test_gpu_models import build, rel  # noqa: E402

EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _edges(name, dev):
    from mmrec_b200.utils import synth
    g = synth.named(name)
    u, i = g.train
    e = torch.stack([torch.from_numpy(u), torch.from_numpy(i) + g.n_users])
    return torch.cat((e, e[[1, 0]]), dim=1).to(dev), g.n_users + g.n_items


def _adj(mode, name, dev):
    from mmrec_b200 import graph
    from mmrec_b200.models.mmgcn import mean_adj_from_edges
    e, n = _edges(name, dev)
    return graph.build_gcn_add_adj(e, n, dev) if mode == "add" else mean_adj_from_edges(e, n)


def _dense64(A):
    r, c, v = A.coo()
    return torch.zeros(A.n_rows, A.n_cols, dtype=torch.float64, device=v.device).index_put_((r, c), v.double(), accumulate=True)


@pytest.mark.parametrize("mode", ["add", "mean"])
def test_two_towers_equal_two_propagations_and_float64(dev, mode):
    from mmrec_b200 import ops
    A = _adj(mode, "small", dev)
    assert A.symmetric == (mode == "add")
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.nn.functional.normalize(torch.randn(A.n_rows, 128, device=dev, generator=g)).requires_grad_(True)
    w = torch.randn(A.n_rows, 128, device=dev, generator=g)
    out = ops.propagate_sum(A, x, 2)
    out.backward(w)
    D = _dense64(A)
    x64, w64 = x.detach().double(), w.double()
    h = D @ x64
    want = (h + x64) + D @ h
    gwant = w64 + D.t() @ (w64 + D.t() @ w64)
    Da, L = D.abs(), int((A.rowptr[1:] - A.rowptr[:-1]).max()) + 2
    bound = 4 * L * EPS32 * (x64.abs() + Da @ x64.abs() + Da @ (Da @ x64.abs()))
    gbound = 4 * L * EPS32 * (w64.abs() + Da.t() @ w64.abs() + Da.t() @ (Da.t() @ w64.abs()))
    assert ((out.detach().double() - want).abs() <= bound).all()
    assert ((x.grad.double() - gwant).abs() <= gbound).all()
    for k in range(2):
        cols = slice(64 * k, 64 * (k + 1))
        xk = x.detach()[:, cols].contiguous().requires_grad_(True)
        o = ops.propagate_sum(A, xk, 2)
        o.backward(w[:, cols].contiguous())
        assert ((out.detach()[:, cols].double() - o.detach().double()).abs() <= 2 * bound[:, cols]).all()
        assert ((x.grad[:, cols].double() - xk.grad.double()).abs() <= 2 * gbound[:, cols]).all()


@pytest.mark.parametrize("mode", ["add", "mean"])
def test_two_towers_exact_operands_bit_for_bit(dev, mode):
    """The adjacency's structure with values in (1/8) Z and x in (1/2) Z: every partial sum is exact in fp32, so the result
    and the gradient equal float64, and each column block the width-64 propagation, bit for bit."""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    A0 = _adj(mode, "tiny", dev)
    r, c, _ = A0.coo()
    key = (r + c) if mode == "add" else (3 * r + c)                     # symmetric values where the matrix is flagged so
    v = (((key % 7) - 3).float() * 0.125)
    A = CSR.from_coo(r, c, v, A0.n_rows, A0.n_cols, sum_duplicates=False, symmetric=A0.symmetric)
    gen = torch.Generator().manual_seed(3)
    x = (torch.randint(-7, 8, (A.n_rows, 128), generator=gen).float() * 0.5).to(dev).requires_grad_(True)
    w = (torch.randint(-3, 4, (A.n_rows, 128), generator=gen).float() * 0.25).to(dev)
    out = ops.propagate_sum(A, x, 2)
    out.backward(w)
    D = _dense64(A)
    x64, w64 = x.detach().double(), w.double()
    h = D @ x64
    assert torch.equal(out.detach().double(), (h + x64) + D @ h)
    assert torch.equal(x.grad.double(), w64 + D.t() @ (w64 + D.t() @ w64))
    for k in range(2):
        cols = slice(64 * k, 64 * (k + 1))
        xk = x.detach()[:, cols].contiguous().requires_grad_(True)
        o = ops.propagate_sum(A, xk, 2)
        o.backward(w[:, cols].contiguous())
        assert torch.equal(out.detach()[:, cols], o.detach()) and torch.equal(x.grad[:, cols], xk.grad)
    again = ops.propagate_sum(A, x.detach(), 2)
    assert torch.equal(again, out.detach())


def _sample(dev, seed=0):
    """An epoch sample of tiny's user graph with some users cut short (padded by repeats) or emptied."""
    from mmrec_b200 import graph
    from mmrec_b200.utils import synth
    d = synth.user_graph_dict(synth.named("tiny"))
    d = {u: [v[0][:(u * 7) % 60], v[1][:(u * 7) % 60]] for u, v in d.items()}
    np.random.seed(seed)
    return graph.UserGraphTable(d, D.K).sample(np.random)


def _reference_aggregation(X, idx, w):
    """`user_rep + User_Graph_sample(user_rep, index, weights)` (dualgnn.py:259-266, 172-173)."""
    return X + torch.matmul(w.unsqueeze(1), X[idx]).squeeze()


def test_user_graph_against_the_reference_expression(dev):
    from mmrec_b200 import graph, ops
    idx, w = _sample(dev)
    G_ = graph.build_user_graph(idx, w, dev)
    it, wt = torch.from_numpy(idx).to(dev), torch.from_numpy(w).to(dev)
    gen = torch.Generator(device=dev).manual_seed(1)
    X = torch.randn(idx.shape[0], 64, device=dev, generator=gen).requires_grad_(True)
    up = torch.randn(idx.shape[0], 64, device=dev, generator=gen)
    out = ops.spmm(G_, X, base=X)
    out.backward(up)
    Xr = X.detach().clone().requires_grad_(True)
    ref = _reference_aggregation(Xr, it, wt)
    ref.backward(up)
    assert rel(out, ref) < 1e-6 and rel(X.grad, Xr.grad) < 1e-6
    assert (out - ref).abs().max().item() < 1e-5 and (X.grad - Xr.grad).abs().max().item() < 1e-5


def test_user_graph_exact_operands_bit_for_bit(dev):
    """Weights in (1/8) Z instead of the softmax, repeated neighbours and users without any: the forward and the backward
    equal float64 and the reference's expression bit for bit."""
    from mmrec_b200 import graph, ops
    idx, w = _sample(dev, seed=4)
    empty = ~w.any(axis=1)
    rng = np.random.default_rng(2)
    w = (rng.integers(-4, 5, w.shape) * 0.125).astype(np.float32)
    w[empty] = 0.0
    w[~empty, 0] = 0.5                                                  # every other user keeps a non-zero row
    assert empty.any() and any(len(set(r)) < D.K for r in idx[~empty])
    G_ = graph.build_user_graph(idx, w, dev)
    it, wt = torch.from_numpy(idx).to(dev), torch.from_numpy(w).to(dev)
    gen = torch.Generator().manual_seed(9)
    X = (torch.randint(-7, 8, (idx.shape[0], 64), generator=gen).float() * 0.5).to(dev).requires_grad_(True)
    up = (torch.randint(-3, 4, (idx.shape[0], 64), generator=gen).float() * 0.25).to(dev)
    out = ops.spmm(G_, X, base=X)
    out.backward(up)
    Xr = X.detach().clone().requires_grad_(True)
    ref = _reference_aggregation(Xr, it, wt)
    ref.backward(up)
    M = torch.zeros(idx.shape[0], idx.shape[0], dtype=torch.float64, device=dev)
    M.index_put_((torch.arange(idx.shape[0], device=dev).repeat_interleave(D.K), it.reshape(-1)), wt.reshape(-1).double(), accumulate=True)
    assert torch.equal(out.detach().double(), X.detach().double() + M @ X.detach().double())
    assert torch.equal(X.grad.double(), up.double() + M.t() @ up.double())
    assert torch.equal(out.detach(), ref.detach()) and torch.equal(X.grad, Xr.grad)


def test_user_graph_memory_at_clothing_shape(dev):
    """40 000 users, 40 neighbours each (a fifth of them padded with repeats), d = 64: the reference gathers a [U, 40, 64]
    fp32 tensor (410 MB) and keeps it for the backward.  The op's peak allocation above what was allocated before it, over
    the forward and the backward, must stay below an eighth of that.  The CSR and its transpose are built first."""
    from mmrec_b200 import graph, ops
    U, k, d = 40000, D.K, 64
    rng = np.random.default_rng(0)
    idx = rng.integers(0, U, (U, k)).astype(np.int64)
    short = rng.random(U) < 0.2
    idx[short, 20:] = idx[short, :20]
    w = torch.softmax(torch.from_numpy(rng.random((U, k)).astype(np.float32)), dim=1).numpy()
    G_ = graph.build_user_graph(idx, w, dev)
    assert G_._t is not None
    X = torch.randn(U, d, device=dev).requires_grad_(True)
    up = torch.randn(U, d, device=dev)
    ops.spmm(G_, X, base=X).backward(up)                                # scratch of this stream and width, once
    X.grad = None
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    out = ops.spmm(G_, X, base=X)
    out.backward(up)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - before
    assert peak < 4 * U * k * d / 8, peak
    del out


# ----------------------------------------------------------------------------------------------------------------------
# the model class against the reference's golden files
# ----------------------------------------------------------------------------------------------------------------------
def _env(text_only):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_")
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, None if text_only else v, t)
    synth.write_user_graph_dict(os.path.join(tmp, "data"), "tiny", g)
    return os.path.join(tmp, "data") + "/"


@pytest.fixture(scope="module")
def env(dev):
    return _env(False)


@pytest.fixture(scope="module")
def env_text(dev):
    return _env(True)


def _sub(gold, p):
    return {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)} if p else {k: gold[k] for k in gold.files}


@pytest.mark.parametrize("p", ["", "text."])
def test_dualgnn_matches_reference(env, env_text, golden, p):
    from mmrec_b200.common.trainer import Trainer
    gold = _sub(golden("dualgnn_tiny.npz"), p)
    config, train, valid, test, model = build("DualGNN", env_text if p else env, {})
    dev = config["device"]
    init = {k[len("init_sha256.param0."):]: str(v) for k, v in gold.items() if k.startswith("init_sha256.")}
    got = {k[len("param0."):]: v for k, v in G.init_digests(model).items()}
    assert got == init, "initial state differs from the reference"       # same keys: a reference state_dict loads strictly
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    assert "result_embed" not in dict(model.named_parameters())
    assert G.sha256_tagged(model.result_embed.cpu().numpy()) == str(gold["result_embed0_sha256"])
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    model.eval()
    with torch.no_grad():
        s0 = model.full_sort_predict(eb)
        assert s0.dtype == torch.float64 and s0.is_cuda
        rows = gold["scores0_rows"]                                     # the reference's CPU product: equal to rounding
        np.testing.assert_allclose(s0[:len(rows)].cpu().numpy(), rows, rtol=1e-12, atol=1e-13)
        idx0 = model.full_sort_topk(eb, 50)
        m = s0.clone()
        m[eb[1][0], eb[1][1]] = -1e10
        assert torch.equal(idx0, torch.topk(m, 50, dim=-1)[1])
    np.random.seed(D.SAMPLE_SEED)
    model.pre_epoch_processing()
    assert G.equal(gold, "sample_idx", model.epoch_user_graph.numpy())
    assert G.equal(gold, "sample_w", model.user_weight_matrix.cpu().numpy())
    seen = {}
    orig = model.user_graph.forward

    def spy(features, user_graph, user_matrix=None, base=None):
        seen["user_rep"] = features.detach()
        return orig(features, user_graph, user_matrix, base=base)
    model.user_graph.forward = spy
    model.train()
    model.zero_grad()
    b = torch.from_numpy(gold["batch"]).to(dev)
    loss = model.calculate_loss(b)
    del model.user_graph.forward
    assert np.array_equal(b.cpu().numpy(), gold["batch_after"])       # the reference's in-place item offset
    for name in ("v_rep", "t_rep"):
        if name + ".sha256" in gold:
            assert G.rel(gold, name, getattr(model, name).detach().squeeze(2).cpu().numpy()) < 1e-5, name
    assert G.rel(gold, "user_rep", seen["user_rep"].cpu().numpy()) < 1e-5
    assert G.rel(gold, "result_embed", model.result_embed.detach().cpu().numpy()) < 1e-5
    loss.backward()
    np.testing.assert_allclose(loss.item(), gold["loss"][0], rtol=1e-5)
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(gold, "grad.")]
    assert set(grads) == {k for k, q in named.items() if q.grad is not None}
    for k in grads:
        assert G.rel(gold, "grad." + k, named[k].grad.cpu().numpy()) < 1e-4, f"grad {k}"
    model.eval()
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        assert s.dtype == torch.float32
        if "scores" in gold:
            assert (s.cpu() - torch.from_numpy(gold["scores"])).abs().max().item() < 1e-5 * np.abs(gold["scores"]).max()
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_dualgnn_topk_equals_mask_topk_of_predict(env):
    from mmrec_b200 import ops
    config, train, valid, test, model = build("DualGNN", env, {})
    dev = config["device"]
    model.pre_epoch_processing()
    model.train()
    model.calculate_loss(next(iter(train)).to(dev)).backward()
    model.eval()
    with torch.no_grad():
        for eb in valid:
            eb = [eb[0].to(dev), eb[1].to(dev)]
            idx = model.full_sort_topk(eb, 50)
            _, want = ops.mask_topk(model.full_sort_predict(eb).clone(), eb[1], 50)
            assert torch.equal(idx, want)


def test_dualgnn_trajectory_replay(env, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches, `np.random` seeded before each epoch's sample:
    per-batch losses and per-epoch metrics."""
    gold = golden("traj_dualgnn_tiny.npz")
    config, train, valid, test, model = build("DualGNN", env, {})
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
        np.random.seed(int(gold["epoch_seed0"]) + ep)
        model.pre_epoch_processing()
        model.train()
        for _ in range(int(nb)):
            trainer.optimizer.zero_grad()
            loss = model.calculate_loss(torch.from_numpy(batches[:, offs[b]:offs[b + 1]].copy()).to(dev))
            np.testing.assert_allclose(loss.item(), gold["losses"][b], rtol=1e-5)
            loss.backward()
            trainer.optimizer.step()
            b += 1
        trainer.lr_scheduler.step()
        v = trainer.evaluate(valid)
        t = trainer.evaluate(test, is_test=True)
        np.testing.assert_allclose([v[k] for k in names], gold["valid"][ep], atol=2e-4)
        np.testing.assert_allclose([t[k] for k in names], gold["test"][ep], atol=2e-4)
    assert b == int(gold["n_steps"])
