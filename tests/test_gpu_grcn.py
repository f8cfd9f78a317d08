"""GRCN on the GPU: the edge-attention kernel (`ops.edge_attention`) against a float64 restatement on power-law graphs at
tiny, baby and clothing shapes (empty rows, rows of one entry, hub rows of thousands, repeated edges, d = 64 / 128 / 80,
tied and large scores) within a stated per-row bound; its backward against float64 autograd through both outputs; its
bits from run to run; a composition of existing ops (kept here only, and by tools/bench_grcn.py) to fp32 reorder error;
the model class against the golden files recorded from the reference (tests/golden/make_golden_grcn.py), two epochs
through FusedAdam, a training step replayed from a CUDA graph, and the peak memory of a training step at clothing's
shape against the reference's expressions on the device."""
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
from make_golden_grcn import CASES, TRAJ_LR, MessagePassing, softmax  # noqa: E402
from test_gpu_models import build  # noqa: E402

U32 = 2.0 ** -24
SHAPES = {"tiny": (300, 120, 1600, 0), "baby": (20000, 7000, 160000, 4000), "clothing": (40000, 23000, 280000, 7000)}


@pytest.fixture(scope="module", autouse=True)
def _leave_no_device_memory():
    """The GPUs are shared, and later files bound their own peak (`tests/test_gpu_spmm_scale.py`): after the last test this
    file releases what it made the process keep -- the library's per-stream scratch, grown here to clothing-scale graphs
    and feature tables (a grown buffer keeps its predecessors alive), and cuBLAS's workspaces, one per stream the file ran
    a matmul on (the CUDA-graph test's side stream adds one).  No CUDA graph of this file outlives its test."""
    yield
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        import gc
        from mmrec_b200 import ops
        gc.collect()
        torch.cuda.synchronize()
        ops._ws_cache.clear()
        torch._C._cuda_clearCublasWorkspaces()
        torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def attention_graph(shape, seed=0, device="cuda"):
    """A GRCN attention CSR over U + I nodes from zipf-popular interactions (repeats kept), with a hub item of `hub` extra
    users, three items and users nobody touches (empty rows) and every degree in between."""
    from mmrec_b200 import graph
    from mmrec_b200.ops import CSR
    n_users, n_items, n_inter, hub = SHAPES[shape]
    rng = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items - 2) ** 0.8
    items = rng.choice(n_items - 3, size=n_inter, p=pop / pop.sum()) + 1
    users = rng.integers(0, n_users - 3, n_inter)
    users = np.concatenate([users, np.arange(hub) % (n_users - 3)])
    items = np.concatenate([items, np.zeros(hub, dtype=np.int64)])
    rows, cols, _ = graph.grcn_edge_order(users, items, n_users, n_items)
    n = n_users + n_items
    return CSR.from_coo(torch.from_numpy(rows).to(device), torch.from_numpy(cols).to(device), None, n, n, sum_duplicates=False)


def features(n, d, kind, seed=1, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    if kind == "ties":                                                # few distinct values: many equal scores in a row
        x = torch.randint(-2, 3, (n, d), generator=g).float() / 4
    else:
        x = torch.randn(n, d, generator=g) / d ** 0.5
        if kind == "large":
            x = x * 6.0
    return x.to(device)


def attention64(A, X, base):
    """The reference's expressions (GATConv + PyG's grouped softmax + 'add') in float64 on the device, differentiable."""
    r, c, _ = A.coo()
    n = A.n_rows
    s = (X[r] * X[c]).sum(1)
    m = torch.full((n,), -float("inf"), dtype=s.dtype, device=s.device).scatter_reduce(0, r, s.detach(), "amax")
    ex = (s - m[r]).exp()
    den = torch.zeros(n, dtype=s.dtype, device=s.device).index_add(0, r, ex) + 1e-16
    alpha = ex / den[r]
    return base + torch.zeros_like(X).index_add(0, r, alpha[:, None] * X[c]), alpha


def compose_attention(A, X, base):
    """The attention as a composition of existing ops (test-only): `sddmm_raw` scores, `torch.segment_reduce` max, the
    exponentials, width-1 K1 row sums and `spmm_values`.  Differentiable w.r.t. X and base (the max detached, as PyG's)."""
    from mmrec_b200 import ops
    r = A.coo()[0]
    deg = (A.rowptr[1:] - A.rowptr[:-1]).to(torch.int64)
    s = ops.sddmm(A, X, X)
    m = torch.segment_reduce(s.detach(), "max", lengths=deg, unsafe=True)
    ex = torch.exp(s - m[r])
    ones = torch.ones(A.n_cols, 1, dtype=torch.float32, device=X.device)
    den = ops.spmm_values(A, ex, ones).reshape(-1) + 1e-16
    alpha = ex / den[r]
    return ops.spmm_values(A, alpha, X) + base, alpha


def _bounds(A, X, Y64, a64, base):
    """Per-entry bound on alpha and per-element bound on Y, from the fp32 error of each row's scores (a dot product of d
    terms: (d + 2) u sum |x_i x_j|), its exponentials, division and sums of deg terms, all with a factor 2 of margin:
      E_i = 2 max_e ds_e + (deg_i + 8) u,  |alpha_e - alpha64_e| <= 2 alpha64_e E_i,
      |Y - Y64|_ik <= 2 (sum_e (|alpha_e - alpha64_e| + (deg_i + 2) u alpha64_e) |X_jk| + 2 u (|base_ik| + |Y64_ik|))."""
    r, c, _ = A.coo()
    n, d = X.shape
    X64 = X.double()
    deg = (A.rowptr[1:] - A.rowptr[:-1]).double()
    ds = (d + 2) * U32 * (X64[r] * X64[c]).abs().sum(1)
    mx = torch.zeros(n, dtype=torch.float64, device=X.device).scatter_reduce(0, r, ds, "amax")
    E = 2 * mx + (deg + 8) * U32
    ea = 2 * a64 * E[r]
    w = ea + (deg[r] + 2) * U32 * a64
    ey = 2 * (torch.zeros_like(X64).index_add(0, r, w[:, None] * X64[c].abs()) + 2 * U32 * (base.double().abs() + Y64.abs()))
    return ea, ey, E, deg


# ------------------------------------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,d,kind", [("tiny", 64, "normal"), ("tiny", 80, "ties"), ("tiny", 128, "large"),
                                          ("baby", 64, "normal"), ("baby", 128, "ties"), ("baby", 80, "large"),
                                          ("clothing", 64, "normal"), ("clothing", 128, "large")])
def test_edge_attention_within_the_per_row_bound_of_float64(dev, shape, d, kind):
    from mmrec_b200 import ops
    A = attention_graph(shape)
    deg = (A.rowptr[1:] - A.rowptr[:-1])
    assert (deg == 0).sum() >= 3 and (deg == 1).any() and int(deg.max()) >= (1000 if shape != "tiny" else 20)
    if shape != "tiny":
        assert ops.edge_attention_heavy_rows(A).numel() > 0                # both routes run
    X = features(A.n_rows, d, kind)
    base = features(A.n_rows, d, "normal", seed=2)
    Y, alpha = ops.edge_attention_raw(A, X, base)
    Y64, a64 = attention64(A, X.double(), base.double())
    ea, ey, E, degd = _bounds(A, X, Y64, a64, base)
    assert ((alpha.double() - a64).abs() <= ea).all()
    assert ((Y.double() - Y64).abs() <= ey).all()
    r = A.coo()[0]
    sums = torch.zeros(A.n_rows, dtype=torch.float64, device=dev).index_add(0, r, alpha.double())
    ne = degd > 0
    tol = torch.zeros_like(sums).index_add(0, r, ea) + (degd + 2) * U32
    assert ((sums[ne] - 1).abs() <= tol[ne]).all()
    assert torch.equal(Y[~ne], base[~ne])                                 # empty rows: Y = base


def test_edge_attention_without_base_and_refusals(dev):
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    A = attention_graph("tiny")
    X = features(A.n_rows, 64, "normal")
    Y, alpha = ops.edge_attention_raw(A, X)
    Yb, alpha_b = ops.edge_attention_raw(A, X, torch.zeros_like(X))
    assert torch.equal(alpha, alpha_b) and torch.equal(Y, Yb)
    with pytest.raises(MMRecError, match="X must be"):
        ops.edge_attention(A, X[:-1])
    with pytest.raises(MMRecError, match="base must be"):
        ops.edge_attention(A, X, X[:, :32].contiguous())
    R = ops.CSR.from_coo(torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev), None, 2, 3)
    with pytest.raises(MMRecError, match="square"):
        ops.edge_attention(R, X[:2])


@pytest.mark.parametrize("shape,d", [("tiny", 64), ("tiny", 80), ("baby", 64), ("baby", 128)])
@pytest.mark.parametrize("through", ["both", "alpha"])
def test_edge_attention_backward_against_float64_autograd(dev, shape, d, through):
    """Gradients of X and base with the upstream gradient arriving through Y and alpha, or through alpha alone (the edge
    weights' path): norm-wise within 1e-4 of float64 autograd (the max detached, as PyG's softmax does)."""
    from mmrec_b200 import ops
    A = attention_graph(shape)
    X0 = features(A.n_rows, d, "normal")
    base0 = features(A.n_rows, d, "normal", seed=2)
    g = torch.Generator().manual_seed(3)
    uY = torch.randn(A.n_rows, d, generator=g).to(dev)
    ua = torch.randn(A.nnz, generator=g).to(dev)
    grads = []
    for fn, dt in ((ops.edge_attention, torch.float32), (attention64, torch.float64)):
        X = X0.to(dt).clone().requires_grad_(True)
        base = base0.to(dt).clone().requires_grad_(True)
        Y, alpha = fn(A, X, base)
        loss = (alpha * ua.to(dt)).sum()
        if through == "both":
            loss = loss + (Y * uY.to(dt)).sum()
        gX, gb = torch.autograd.grad(loss, (X, base), allow_unused=True)
        grads.append((gX, gb))
    (gX, gb), (gX64, gb64) = grads
    assert (gX.double() - gX64).norm().item() <= 1e-4 * gX64.norm().item()
    if through == "both":
        assert torch.equal(gb.double(), gb64)
    else:
        assert gb is None or not gb.any()


def test_edge_attention_repeats_its_bits(dev):
    from mmrec_b200 import ops
    A = attention_graph("baby")
    X0 = features(A.n_rows, 64, "normal")
    g = torch.Generator().manual_seed(3)
    uY = torch.randn(A.n_rows, 64, generator=g).to(dev)
    ua = torch.randn(A.nnz, generator=g).to(dev)
    runs = []
    for _ in range(2):
        X = X0.clone().requires_grad_(True)
        Y, alpha = ops.edge_attention(A, X, base=X)
        (gX,) = torch.autograd.grad((Y * uY).sum() + (alpha * ua).sum(), (X,))
        runs.append((Y, alpha, gX))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("shape,d", [("tiny", 64), ("baby", 64), ("baby", 128), ("clothing", 64)])
def test_edge_attention_agrees_with_the_composition_of_existing_ops(dev, shape, d):
    from mmrec_b200 import ops
    A = attention_graph(shape)
    X0 = features(A.n_rows, d, "normal")
    g = torch.Generator().manual_seed(4)
    uY = torch.randn(A.n_rows, d, generator=g).to(dev)
    outs = []
    for fn in (ops.edge_attention, compose_attention):
        X = X0.clone().requires_grad_(True)
        Y, alpha = fn(A, X, X)
        (gX,) = torch.autograd.grad((Y * uY).sum(), (X,))
        outs.append((Y.detach(), alpha.detach(), gX))
    (Y, a, gX), (Yc, ac, gXc) = outs
    Y64, a64 = attention64(A, X0.double(), X0.double())
    ea, _, _, _ = _bounds(A, X0, Y64, a64, X0)
    assert ((a.double() - ac.double()).abs() <= 2 * ea).all()
    assert (Y - Yc).norm().item() <= 1e-5 * Yc.norm().item()
    assert (gX - gXc).norm().item() <= 1e-4 * gXc.norm().item()


# ------------------------------------------------------------------------------------------------------------------------
# the reference's expressions on the device (the generator's PyG shim), for the memory comparison and tools/bench_grcn.py
# ------------------------------------------------------------------------------------------------------------------------
class _GATConv(MessagePassing):
    """`GATConv.message` (src/models/grcn.py:61-73)."""

    def message(self, x_i, x_j, size_i, edge_index_i):
        self.alpha = softmax(torch.mul(x_i, x_j).sum(dim=-1), edge_index_i, num_nodes=size_i)
        return x_j * self.alpha.view(-1, 1)


class _SAGEConv(MessagePassing):
    """`SAGEConv.message` (src/models/grcn.py:32-37)."""

    def forward(self, x, edge_index, weight_vector):
        self.weight_vector = weight_vector
        return self.propagate(edge_index, x=x)

    def message(self, x_j):
        return x_j * self.weight_vector


def reference_loss(model, batch):
    """`GRCN.forward` + `calculate_loss` (src/models/grcn.py:139-166, 224-333) on the device from the model's own
    parameters: the [2E, d] gathers, messages and `index_add_` scatters of PyG's message passing, routing loop included."""
    U = model.n_users
    ei = model.edge_index
    sym = torch.cat((ei, ei[[1, 0]]), dim=1)
    reps, ws = [], []
    for gcn in [model.v_gcn] + ([model.t_gcn] if model.t_feat is not None else []):
        features = F.normalize(F.leaky_relu(F.linear(gcn.features, gcn.MLP.weight, gcn.MLP.bias)))
        preference = F.normalize(gcn.preference)
        conv = _GATConv()
        for _ in range(gcn.num_routing):
            x_hat_1 = conv.propagate(ei, x=torch.cat((preference, features), dim=0))
            preference = F.normalize(preference + x_hat_1[:U])
        x = torch.cat((preference, features), dim=0)
        reps.append(x + conv.propagate(sym, x=x))
        ws.append(conv.alpha.view(-1, 1))
    conf = torch.cat((model.model_specific_conf[ei[0]], model.model_specific_conf[ei[1]]), dim=0)
    weight = torch.relu(torch.max(torch.cat(ws, dim=1) * conf, dim=1)[0].view(-1, 1))
    x = F.normalize(model.id_gcn.id_embedding)
    sage = _SAGEConv()
    x1 = sage(x, sym, weight)
    out = torch.cat([x + x1 + sage(x1, sym, weight)] + reps, dim=1)
    user_tensor = batch[0].repeat_interleave(2)
    item_tensor = torch.stack((batch[1] + U, batch[2] + U)).t().contiguous().view(-1)
    score = torch.sum(out[user_tensor] * out[item_tensor], dim=1).view(-1, 2)
    loss = -torch.mean(torch.log(torch.sigmoid(torch.matmul(score, model.weight))))
    reg = (model.id_gcn.id_embedding[user_tensor] ** 2 + model.id_gcn.id_embedding[item_tensor] ** 2).mean()
    reg = reg + (model.v_gcn.preference ** 2).mean() + (model.v_gcn.preference[user_tensor] ** 2).mean()
    if model.t_feat is not None:
        reg = reg + (model.t_gcn.preference[user_tensor] ** 2).mean()
    return loss + model.reg_weight * reg


# ------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------
def make_env(shape, mods, seed=0):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_grcn_")
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
    return {m: make_env("tiny", m) for m in ("vt", "v")}


def _sub(gold, p):
    return {k[len(p):]: gold[k] for k in gold.files
            if k.startswith(p) and not any(k.startswith(q) for q in CASES if q and q != p and len(q) > len(p))}


def _check_topk(gold, s, eb, idx):
    want = torch.from_numpy(gold["topk50"]).long()
    m = s.clone()
    m[eb[1][0], eb[1][1]] = -1e10
    m = m.cpu().double()
    scale = m[m > -1e9].abs().max().item()
    diff = idx.cpu() != want
    gap = (m.gather(1, idx.cpu()) - m.gather(1, want)).abs()
    assert (gap[diff] <= 1e-5 * scale).all() and diff.float().mean().item() < 0.05


@pytest.mark.parametrize("p", list(CASES))
def test_grcn_matches_reference(envs, golden, p):
    from mmrec_b200.common.trainer import Trainer
    full = golden("grcn_tiny.npz")
    gold = _sub(full, p)
    config, train, valid, test, model = build("GRCN", envs[CASES[p][1]], dict(CASES[p][0]))
    dev = config["device"]
    init = {k[len("init_sha256."):]: str(v) for k, v in gold.items() if k.startswith("init_sha256.")}
    assert G.init_digests(model) == init, "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    model.eval()
    with torch.no_grad():                                              # before training: the random `result`
        assert G.rel(gold, "pre.scores", model.full_sort_predict(eb).cpu().numpy()) < 1e-5
    seen = {}
    orig = model.edge_weight

    def spy(alphas):
        w = orig(alphas)
        seen["alphas"], seen["weight"] = [a.detach().reshape(-1) for a in alphas], w.detach()
        return w
    model.edge_weight = spy
    model.train()
    model.zero_grad(set_to_none=True)
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    del model.edge_weight
    order = model.edge_order.cpu().numpy()
    for name, a in zip(("alpha_v", "alpha_t"), seen["alphas"]):
        want = gold[name][order].reshape(-1)
        np.testing.assert_allclose(a.cpu().numpy(), want, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(seen["weight"].cpu().numpy(), gold["weight"][order], rtol=1e-5, atol=1e-7)
    assert G.rel(gold, "representation", model.result.detach().cpu().numpy()) < 1e-5
    loss.backward()
    assert tuple(loss.shape) == tuple(gold["loss_shape"])
    np.testing.assert_allclose(loss.item(), gold["loss"][0], rtol=1e-5)
    named = dict(model.named_parameters())
    rec = [k[len("grad."):] for k in G.recorded(gold, "grad.")]
    assert set(rec) == {k for k, q in named.items() if q.grad is not None}
    for k in rec:
        assert G.rel(gold, "grad." + k, named[k].grad.cpu().numpy()) < 1e-4, f"grad {k}"
    model.zero_grad(set_to_none=True)
    model.eval()
    with torch.no_grad():                                              # after one batch: that batch's representation
        s = model.full_sort_predict(eb)
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
        _check_topk(gold, s, eb, model.full_sort_topk(eb, 50))
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_grcn_trajectory_through_fused_adam(envs, golden):
    gold = golden("traj_grcn_tiny.npz")
    config, train, valid, test, model = build("GRCN", envs["vt"], {"learning_rate": TRAJ_LR})
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
    for k, q in model.state_dict().items():
        want = gold["final." + k]
        assert np.linalg.norm(q.cpu().numpy() - want) <= 1e-4 * max(np.linalg.norm(want), 1e-30), k


def test_training_step_replayed_from_a_cuda_graph_gives_the_eager_bits(envs, golden):
    """`calculate_loss` + `backward` captured once on a side stream and replayed: the loss, `result` and every gradient
    equal an eager step's bits on the same batch."""
    gold = golden("grcn_tiny.npz")
    config, train, valid, test, model = build("GRCN", envs["vt"], {})
    dev = config["device"]
    model.train()
    static = torch.from_numpy(gold["batch"]).to(dev)
    params = [q for q in model.parameters() if q.requires_grad]

    def step():
        loss = model.calculate_loss(static)
        loss.backward()
        return loss

    def snapshot(loss):
        return [loss.detach().clone(), model.result.detach().clone()] + [q.grad.clone() for q in params]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            model.zero_grad(set_to_none=True)
            step()
    torch.cuda.synchronize()
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        loss_c = step()
    torch.cuda.synchronize()
    runs = []
    for _ in range(2):
        for q in params:
            q.grad.zero_()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            g.replay()
        torch.cuda.synchronize()
        runs.append(snapshot(loss_c))
    for q in params:
        q.grad = None
    with torch.cuda.stream(side):
        eager = snapshot(step())
    torch.cuda.synchronize()
    for run in runs:
        for a, e in zip(run, eager):
            assert torch.equal(a, e)


def test_training_step_at_clothing_shape_peaks_below_the_reference_expressions(dev):
    """Peak memory above the model of `calculate_loss` + backward at clothing's shape (63 000 nodes, 2 x 224 000 edges,
    features F = 4096 and 384), the model against the reference's message passing on the device (`reference_loss`): the
    reference gathers x_i, x_j and the messages as [2E, d] tensors for each modality and convolution."""
    config, train, valid, test, model = build("GRCN", make_env("clothing", "vt"), {"train_batch_size": 2048})
    batch = next(iter(train)).to(config["device"])
    model.train()
    peaks = {}
    for name, fn in (("model", model.calculate_loss), ("reference", lambda b: reference_loss(model, b))):
        model.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(batch).sum().backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    print(f"GRCN clothing step peak above the model: {peaks['model'] / 2**20:.0f} MiB, reference expressions "
          f"{peaks['reference'] / 2**20:.0f} MiB, ratio {peaks['reference'] / peaks['model']:.2f}")
    assert peaks["model"] < peaks["reference"]
