"""VBPR and BPR on the GPU: the loss kernel (`ops.bpr_mf_loss`, csrc/mf_bpr.cu) forward and backward against the torch
expression on the device -- bit for bit on exactly representable inputs, where the dots and norms are exact and every
element-wise step must round as autograd's does, and against float64 within a stated per-row bound on random inputs --
over repeated and unsorted indices, B = 1, B past two sweeps of the grid, zero matrices (norm 0), NaN rows, dp = 0 and
dp > 0; its bits from run to run; the model classes against the golden files recorded from the reference
(tests/golden/make_golden_vbpr.py) and both trajectories through FusedAdam; `full_sort_topk` against the mask and top-k
of `full_sort_predict`; the gathered route's gradients against the reference's full-table expression; a training step
replayed from a CUDA graph; and the peak memory of a training step at clothing's shape."""
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

import golden_io as G  # noqa: E402
import vbpr_golden as V  # noqa: E402
from test_gpu_models import build  # noqa: E402

U32 = 2.0 ** -24


@pytest.fixture(scope="module", autouse=True)
def _leave_no_device_memory():
    """The GPUs are shared, and later files bound their own peak: after the last test this file releases what it made the
    process keep -- the library's per-stream scratch (a grown buffer keeps its predecessors alive) and cuBLAS's
    workspaces, one per stream the file ran a matmul on.  No CUDA graph of this file outlives its test."""
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


# ------------------------------------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------------------------------------
def kernel_rows(U, A, P, users, pos, neg, rw, g):
    """The raw entry points: (loss, x, norms, gU rows, gA rows, gP rows) for the upstream gradient g (one fp32)."""
    from mmrec_b200 import _lib, ops
    lib = _lib.load()
    B, du, da = users.numel(), U.shape[1], A.shape[1]
    dp = 0 if P is None else P.shape[1]
    loss, x, norms = (torch.empty(n, device=U.device) for n in (1, B, 3))
    ws = torch.empty(lib.mmrec_bpr_mf_workspace_bytes(B), dtype=torch.uint8, device=U.device)
    ops.check(lib.mmrec_bpr_mf_f32(B, du, da, dp, U.data_ptr(), A.data_ptr(), ops._ptr(P), users.data_ptr(), pos.data_ptr(),
                                   neg.data_ptr(), rw, loss.data_ptr(), x.data_ptr(), norms.data_ptr(), ws.data_ptr(), ws.numel(),
                                   ops._stream()), "bpr_mf")
    gU, gA = torch.empty(B, du, device=U.device), torch.empty(2 * B, da, device=U.device)
    gP = None if P is None else torch.empty(2 * B, dp, device=U.device)
    ops.check(lib.mmrec_bpr_mf_bwd_f32(B, du, da, dp, U.data_ptr(), A.data_ptr(), ops._ptr(P), users.data_ptr(), pos.data_ptr(),
                                       neg.data_ptr(), rw, x.data_ptr(), norms.data_ptr(), g.data_ptr(), gU.data_ptr(), gA.data_ptr(),
                                       ops._ptr(gP), ops._stream()), "bpr_mf_bwd")
    return loss, x, norms, gU, gA, gP


def torch_rows(U, A, P, users, pos, neg, rw, g, dtype=torch.float32):
    """The reference's expression with the gathered matrices as leaves: (loss, x, norms, gU rows, [gPos; gNeg] rows)."""
    B = users.numel()
    ue = U[users].to(dtype).requires_grad_(True)
    pe, ne = A[pos], A[neg]
    if P is not None:
        pe, ne = torch.cat((pe, P[:B]), -1), torch.cat((ne, P[B:]), -1)
    pe, ne = pe.to(dtype).requires_grad_(True), ne.to(dtype).requires_grad_(True)
    ps, ns = torch.mul(ue, pe).sum(dim=1), torch.mul(ue, ne).sum(dim=1)
    from mmrec_b200.common.loss import BPRLoss, EmbLoss
    loss = BPRLoss()(ps, ns) + rw * EmbLoss()(ue, pe, ne)
    loss.backward(g.to(dtype))
    norms = torch.stack([torch.norm(t.detach()) for t in (ue, pe, ne)])
    return loss.detach(), (ps - ns).detach(), norms, ue.grad, torch.cat((pe.grad, ne.grad))


def _split(gI, da):
    return gI[:, :da], gI[:, da:]


def same_bits(a, b):
    """Equal bits, except that NaN equals NaN (torch's and the kernel's NaNs need not share a payload)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def operands(dev, n_users, n_items, B, da, dp, idx_kind, exact, seed=0):
    g = torch.Generator().manual_seed(seed)
    if exact:                                         # multiples of 1/4 in [-1/2, 1/2]: dots and sums of squares are exact
        def mk(*s):
            return (torch.randint(-2, 3, s, generator=g).float() / 4)
    else:
        def mk(*s):
            return torch.randn(*s, generator=g) * 0.1
    U, A = mk(n_users, da + dp), mk(n_items, da)
    P = mk(2 * B, dp) if dp else None
    if idx_kind == "repeat":                          # few distinct rows, unsorted, pos and neg sharing items
        users = torch.randint(0, min(n_users, 5), (B,), generator=g)
        pos = torch.randint(0, min(n_items, 4), (B,), generator=g)
        neg = torch.randint(0, min(n_items, 4), (B,), generator=g)
    else:
        users = torch.randint(0, n_users, (B,), generator=g)
        pos, neg = torch.randint(0, n_items, (B,), generator=g), torch.randint(0, n_items, (B,), generator=g)
    return [t.to(dev) for t in (U, A)] + [None if P is None else P.to(dev)] + [t.to(dev) for t in (users, pos, neg)]


# (B, da, dp, idx kind): BPR's 64 + 0 and VBPR's 64 + 64 (vectorised), odd widths on the scalar path, B = 1, and B past two
# sweeps of the grid (8 warps x 8 CTAs per SM)
KERNEL_CASES = [(1, 64, 0, "random"), (1, 64, 64, "random"), (37, 64, 0, "repeat"), (300, 64, 64, "repeat"),
                (300, 64, 64, "random"), (300, 24, 13, "random"), (97, 33, 0, "repeat"), (300, 32, 32, "random"),
                (20000, 64, 0, "random"), (20000, 64, 64, "repeat")]


@pytest.mark.parametrize("B,da,dp,idx_kind", KERNEL_CASES)
def test_kernel_equals_the_torch_expression_bit_for_bit_on_exact_inputs(dev, B, da, dp, idx_kind):
    U, A, P, users, pos, neg = operands(dev, 500, 400, B, da, dp, idx_kind, exact=True)
    rw, g = 2.0, torch.tensor([0.75], device=dev)
    k_loss, k_x, k_n, k_gU, k_gA, k_gP = kernel_rows(U, A, P, users, pos, neg, rw, g)
    t_loss, t_x, t_n, t_gU, t_gI = torch_rows(U, A, P, users, pos, neg, rw, g)
    assert torch.equal(k_x, t_x) and torch.equal(k_n, t_n)
    ta, tp = _split(t_gI, da)
    assert torch.equal(k_gU, t_gU)
    assert torch.equal(k_gA, ta)
    assert (k_gP is None and dp == 0) or torch.equal(k_gP, tp)
    # the loss sums B inexact log terms: the order of that sum is the kernel's own
    assert abs(k_loss.item() - t_loss.item()) <= 4 * U32 * (B + 8) * (abs(t_loss.item()) + 1.0)


@pytest.mark.parametrize("dp", [0, 64])
@pytest.mark.parametrize("special", ["zero_users", "zero_all", "nan_row"])
def test_zero_matrices_and_nan_rows_follow_the_torch_expression(dev, dp, special):
    """A zero U_b (norm 0: autograd's masked_fill gives a 0, not a NaN), all three zero (B = 1, x = 0), and a NaN item row."""
    B = 1 if special == "zero_all" else 50
    U, A, P, users, pos, neg = operands(dev, 60, 40, B, 64, dp, "random", exact=True, seed=3)
    if special in ("zero_users", "zero_all"):
        U[users] = 0.0
    if special == "zero_all":
        A[pos] = 0.0
        A[neg] = 0.0
        if P is not None:
            P.zero_()
    if special == "nan_row":
        A[pos[7]] = float("nan")
    g = torch.tensor([1.0], device=dev)
    k = kernel_rows(U, A, P, users, pos, neg, 0.5, g)
    t = torch_rows(U, A, P, users, pos, neg, 0.5, g)
    assert same_bits(k[1], t[1]) and same_bits(k[2], t[2])
    assert same_bits(k[3], t[3])
    ta, tp = _split(t[4], 64)
    assert same_bits(k[4], ta) and (dp == 0 or same_bits(k[5], tp))
    if special == "nan_row":
        assert torch.isnan(k[0]).all()
    elif special == "zero_all":                                          # B = 1: no sum to order
        assert same_bits(k[0], t[0])
        assert (k[3] == 0).all() and (k[4] == 0).all()
    else:
        assert abs(k[0].item() - t[0].item()) <= 4 * U32 * (B + 8) * (abs(t[0].item()) + 1.0)


@pytest.mark.parametrize("B,da,dp", [(1, 64, 64), (512, 64, 0), (2048, 64, 64), (3000, 40, 24), (20000, 64, 64)])
def test_kernel_within_the_per_row_bound_of_float64(dev, B, da, dp):
    """x_b and every gradient row against float64 autograd.  Per row, with u = 2^-24 and du = da + dp:
      |x - x64| <= 2 (du + 6) u (sum|u p| + sum|u n|) = Dx,
      |gx - gx64| <= |g| / (4B) Dx + 8 u |gx64|  (the loss's slope in x is at most |g| / (4B)) = Dgx,
    and for each element of a gradient row, with the norm term q = gn x / ||.|| and the kernel's relative norm error e:
      |gU - gU64| <= 2 (Dgx (|p| + |n|) + (e + 4 u) |q64| + 4 u (|q64| + |gx64| (|p| + |n|))),  likewise for the item rows."""
    U, A, P, users, pos, neg = operands(dev, 3000, 2000, B, da, dp, "random", exact=False, seed=B)
    rw, g = 0.01, torch.tensor([1.0], device=dev)
    k_loss, k_x, k_n, k_gU, k_gA, k_gP = kernel_rows(U, A, P, users, pos, neg, rw, g)
    t_loss, t_x, t_n, t_gU, t_gI = torch_rows(U, A, P, users, pos, neg, rw, g, dtype=torch.float64)
    du = da + dp
    ue = U[users].double()
    pe, ne = A[pos].double(), A[neg].double()
    if P is not None:
        pe, ne = torch.cat((pe, P[:B].double()), -1), torch.cat((ne, P[B:].double()), -1)
    Dx = 2 * (du + 6) * U32 * ((ue * pe).abs().sum(1) + (ue * ne).abs().sum(1))
    assert ((k_x.double() - t_x).abs() <= Dx).all()
    e = ((k_n.double() - t_n).abs() / t_n).max().item()
    assert e <= (B * du + 64) * U32                                      # any summation order of B du squares
    s = torch.sigmoid(t_x)
    gx64 = -(1.0 / B) * (1 - s) * s / (s + 1e-10)
    Dgx = 1.0 / (4 * B) * Dx + 8 * U32 * gx64.abs()
    gn = rw / B

    def bound(x_rows, q_norm, other_abs, dgx, gxa):
        q = (gn * x_rows / q_norm).abs()
        return 2 * (dgx[:, None] * other_abs + (e + 4 * U32) * q + 4 * U32 * (q + gxa[:, None] * other_abs))
    assert ((k_gU.double() - t_gU).abs() <= bound(ue, t_n[0], pe.abs() + ne.abs(), Dgx, gx64.abs())).all()
    k_gI = torch.cat((torch.cat((k_gA[:B], k_gP[:B]), -1), torch.cat((k_gA[B:], k_gP[B:]), -1))) if dp else k_gA
    norms = torch.cat((t_n[1].expand(B), t_n[2].expand(B)))[:, None]
    two = (torch.cat((Dgx, Dgx)), torch.cat((gx64, gx64)).abs())
    assert ((k_gI.double() - t_gI).abs() <= bound(torch.cat((pe, ne)), norms, torch.cat((ue, ue)).abs(), *two)).all()
    assert abs(k_loss.item() - t_loss.item()) <= 8 * U32 * (B + 8 * du) * (abs(t_loss.item()) + 1.0)


def test_op_gives_the_same_bits_on_every_run_and_scatters_the_tables(dev):
    """`ops.bpr_mf_loss` twice on repeated, unsorted indices: the same loss and table gradients, bit for bit; the table
    gradients equal `index_add_` of the kernel's rows to fp32 reorder error."""
    from mmrec_b200 import ops
    U, A, P, users, pos, neg = operands(dev, 50, 30, 4000, 64, 64, "repeat", exact=False, seed=9)
    runs = []
    for _ in range(2):
        Ul, Al, Pl = (t.clone().requires_grad_(True) for t in (U, A, P))
        loss = ops.bpr_mf_loss(Ul, Al, Pl, users, pos, neg, 0.1)
        loss.backward()
        runs.append((loss.detach(), Ul.grad, Al.grad, Pl.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    _, _, _, gU, gA, gP = kernel_rows(U, A, P, users, pos, neg, 0.1, torch.ones(1, device=dev))
    assert torch.equal(runs[0][3], gP)
    ref_u = torch.zeros_like(U).index_add_(0, users, gU)
    ref_a = torch.zeros_like(A).index_add_(0, torch.cat((pos, neg)), gA)
    assert torch.allclose(runs[0][1], ref_u, rtol=1e-5, atol=1e-7) and torch.allclose(runs[0][2], ref_a, rtol=1e-5, atol=1e-7)
    assert tuple(runs[0][0].shape) == (1,)


# ------------------------------------------------------------------------------------------------------------------------
# the models
# ------------------------------------------------------------------------------------------------------------------------
def make_env(shape, mods):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_vbpr_")
    u, i, e, d, f = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    if shape == "tiny":
        v, t = synth.make_features(i, f, seed=1)
    else:
        rng = np.random.default_rng(1)
        v, t = rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", gr, v if "v" in mods else None, t if "t" in mods else None)
    return os.path.join(tmp, "data") + "/"


@pytest.fixture(scope="module")
def envs(dev):
    return {m: make_env("tiny", m) for m in ("vt", "t", "v", "")}


def _sub(gold, p):
    return {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)}


def _case(golden, p):
    name, mods = V.CASES[p]
    return name, mods, _sub(golden(f"{name.lower()}_tiny.npz"), p)


def _check_topk(gold, s, eb, idx):
    want = torch.from_numpy(gold["topk50"]).long()
    m = s.clone()
    m[eb[1][0], eb[1][1]] = -1e10
    m = m.cpu().double()
    scale = m[m > -1e9].abs().max().item()
    diff = idx.cpu() != want
    gap = (m.gather(1, idx.cpu()) - m.gather(1, want)).abs()
    assert (gap[diff] <= 1e-5 * scale).all() and diff.float().mean().item() < 0.05


@pytest.mark.parametrize("p", list(V.CASES))
def test_model_matches_reference(envs, golden, p):
    from mmrec_b200.common.trainer import Trainer
    name, mods, gold = _case(golden, p)
    config, train, valid, test, model = build(name, envs[mods], {})
    dev = config["device"]
    init = {k[len("init_sha256."):]: str(v) for k, v in gold.items() if k.startswith("init_sha256.")}
    assert G.init_digests(model) == init, "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    model.train()
    model.zero_grad(set_to_none=True)
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
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
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
        _check_topk(gold, s, eb, model.full_sort_topk(eb, 50))
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


@pytest.mark.parametrize("name", list(V.TRAJ))
def test_trajectory_through_fused_adam(envs, golden, name):
    """Two epochs on the recorded batches: every loss, the per-epoch metrics and the final state; and no training step
    draws from torch's CPU or device generator (the reference's `F.dropout(·, 0.0)` draws nothing either)."""
    gold = golden(f"traj_{name.lower()}_tiny.npz")
    config, train, valid, test, model = build(name, envs[V.TRAJ[name]], {})
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches = gold["batches"]
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    assert bool(np.all(gold["rng_kept"]))
    b = 0
    for ep, nb in enumerate(gold["batches_per_epoch"]):
        model.pre_epoch_processing()
        model.train()
        for _ in range(int(nb)):
            cpu_rng, dev_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
            trainer.optimizer.zero_grad()
            loss = model.calculate_loss(torch.from_numpy(batches[:, offs[b]:offs[b + 1]].copy()).to(dev))
            np.testing.assert_allclose(loss.item(), gold["losses"][b], rtol=1e-5)
            loss.backward()
            trainer.optimizer.step()
            assert torch.equal(cpu_rng, torch.get_rng_state()) and torch.equal(dev_rng, torch.cuda.get_rng_state())
            b += 1
        trainer.lr_scheduler.step()
        v = trainer.evaluate(valid)
        t = trainer.evaluate(test, is_test=True)
        np.testing.assert_allclose([v[k] for k in names], gold["valid"][ep], atol=2e-4)
        np.testing.assert_allclose([t[k] for k in names], gold["test"][ep], atol=2e-4)
    assert b == int(gold["n_steps"])
    for k, q in model.state_dict().items():
        assert G.rel(gold, "final." + k, q.cpu().numpy()) < 1e-4, k


@pytest.mark.parametrize("p", list(V.CASES))
def test_topk_equals_mask_topk_of_predict(envs, golden, p):
    from mmrec_b200 import ops
    name, mods, gold = _case(golden, p)
    config, train, valid, test, model = build(name, envs[mods], {})
    dev = config["device"]
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        _, want = ops.mask_topk(s.clone(), eb[1], 50)
        got = model.full_sort_topk(eb, 50)
    m = s.clone()
    m[eb[1][0], eb[1][1]] = -1e10
    diff = got != want
    gap = (m.gather(1, got) - m.gather(1, want)).abs()
    assert (gap[diff] <= 1e-6 * m[m > -1e9].abs().max()).all()


def reference_loss(model, interaction):
    """The reference's `forward` + `calculate_loss` (src/models/vbpr.py:69-98, bpr.py:62-86) on the device: VBPR's
    full-table `nn.Linear` of the raw table and its concatenation with the ID table, then the gathers and the torch loss."""
    if hasattr(model, "item_linear"):
        user_embeddings = model.u_embedding
        item_embeddings = torch.cat((model.i_embedding, model.item_linear(model.item_raw_features)), -1)
    else:
        user_embeddings, item_embeddings = model.user_embedding.weight, model.item_embedding.weight
    user_e = user_embeddings[interaction[0], :]
    pos_e, neg_e = item_embeddings[interaction[1], :], item_embeddings[interaction[2], :]
    pos_item_score, neg_item_score = torch.mul(user_e, pos_e).sum(dim=1), torch.mul(user_e, neg_e).sum(dim=1)
    return model.loss(pos_item_score, neg_item_score) + model.reg_weight * model.reg_loss(user_e, pos_e, neg_e)


@pytest.mark.parametrize("p", list(V.CASES))
def test_gathered_training_route_equals_the_full_table_expression(envs, golden, p):
    """The model's loss and every gradient -- the projection's weight and bias over the 2B gathered rows included --
    against the reference's full-table route on the device, each gradient within 1e-5 of the largest one's scale."""
    name, mods, gold = _case(golden, p)
    config, train, valid, test, model = build(name, envs[mods], {})
    batch = torch.from_numpy(gold["batch"]).to(config["device"])
    model.train()
    out = {}
    for route, fn in (("model", model.calculate_loss), ("reference", lambda b: reference_loss(model, b))):
        model.zero_grad(set_to_none=True)
        loss = fn(batch)
        loss.backward()
        out[route] = (loss.item(), {k: q.grad.clone() for k, q in model.named_parameters()})
    assert abs(out["model"][0] - out["reference"][0]) <= 1e-6 * abs(out["reference"][0])
    scale = max(r.norm().item() for r in out["reference"][1].values())
    for k, r in out["reference"][1].items():
        got = out["model"][1][k]
        assert (got - r).norm().item() <= 1e-5 * max(r.norm().item(), 1e-3 * scale), k


@pytest.mark.parametrize("p", ["vt.", "bpr."])
def test_training_step_replayed_from_a_cuda_graph_gives_the_eager_bits(envs, golden, p):
    """`calculate_loss` + `backward` captured once on a side stream and replayed: the loss and every gradient equal an
    eager step's bits on the same batch."""
    name, mods, gold = _case(golden, p)
    config, train, valid, test, model = build(name, envs[mods], {})
    dev = config["device"]
    model.train()
    static = torch.from_numpy(gold["batch"]).to(dev)
    params = [q for q in model.parameters() if q.requires_grad]

    def step():
        loss = model.calculate_loss(static)
        loss.backward()
        return loss

    def snapshot(loss):
        return [loss.detach().clone()] + [q.grad.clone() for q in params]

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
    del g
    for run in runs:
        for a, e in zip(run, eager):
            assert torch.equal(a, e)


def test_training_step_at_clothing_shape_peaks_below_the_reference_expressions(dev):
    """Peak memory above the model of VBPR's `calculate_loss` + backward at clothing's shape (23 000 items, raw table
    4480 wide, B = 2048): the model projects 2B rows, the reference's expressions the whole table.  Each route is
    measured on its second step: the first one grows the library's per-stream scratch (K2's and K5's), which every later
    step reuses."""
    config, train, valid, test, model = build("VBPR", make_env("clothing", "vt"), {"train_batch_size": 2048})
    batch = next(iter(train)).to(config["device"])
    model.train()
    peaks = {}
    for name, fn in (("model", model.calculate_loss), ("reference", lambda b: reference_loss(model, b))):
        model.zero_grad(set_to_none=True)
        fn(batch).sum().backward()
        model.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(batch).sum().backward()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    print(f"VBPR clothing step peak above the model: {peaks['model'] / 2**20:.0f} MiB, reference expressions "
          f"{peaks['reference'] / 2**20:.0f} MiB, ratio {peaks['reference'] / peaks['model']:.2f}")
    assert peaks["model"] < peaks["reference"]
