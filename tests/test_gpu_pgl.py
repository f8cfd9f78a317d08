"""PGL on the GPU: the loss op (`ops.pgl_loss`, csrc/pgl_loss.cu with K8 for the B x B sums) forward and backward against
the torch expression on the device -- bit for bit on exactly representable inputs (every dot, norm and normalised entry
exact) at reg_weight 0, the loss to the batch sum's order and the gradients to a stated bound at reg_weight > 0 (there
the gradient passes through K8's sums and F.normalize's row sum of them) -- and against float64 within a per-row bound on
random inputs; zero and NaN rows; its bits from run to run; the dropout scales torch uses; the device generator after a
training step against the reference's expressions; the model against every golden case (recorded keep indices and
masks); two epochs through FusedAdam; `full_sort_topk`; a CUDA-graph replay; and peak memory at clothing's shape."""
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
import pgl_golden as P  # noqa: E402
from test_gpu_models import build  # noqa: E402

U32 = 2.0 ** -24


@pytest.fixture(scope="module", autouse=True)
def _leave_no_device_memory():
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
# the op
# ------------------------------------------------------------------------------------------------------------------------
def k8_ttl(v1, v2, tau):
    from mmrec_b200 import ops
    return ops.expsum_rows(v1, v2, tau)


def run_op(UA, IA, users, pos, neg, masks, p, rw):
    from mmrec_b200 import ops
    UA, IA = UA.clone().requires_grad_(True), IA.clone().requires_grad_(True)
    loss = ops.pgl_loss(UA, IA, users, pos, neg, masks, p, rw)
    loss.backward()
    return loss.detach(), UA.grad, IA.grad


def run_torch(UA, IA, users, pos, neg, masks, p, rw, dtype=torch.float32, k8=True):
    """The reference's expression on the device, the dropout as torch's device kernels round it, and (k8) K8 for the
    [B, B] exp-sums."""
    UA, IA = UA.to(dtype).requires_grad_(True), IA.to(dtype).requires_grad_(True)
    loss = P.torch_pgl_loss(UA, IA, users, pos, neg, masks, p, rw, drop=P.device_drop, ttl_fn=k8_ttl if k8 else None)
    loss.backward()
    return loss.detach(), UA.grad, IA.grad


def exact_operands(dev, B, seed=0):
    """Unique users and items; every row 16 entries of +-1/4; masks keeping all 16 of u and p for the views a and c and
    exactly 4 for b and d (random elsewhere): at p = 0.2 the views' norms are 1.25 and 0.625, every normalised entry and
    every dot exact."""
    g = torch.Generator().manual_seed(seed)
    D = 128
    n_users, n_items = B + 3, 2 * B + 5
    UA, IA = torch.zeros(n_users, D), torch.zeros(n_items, D)
    sup_u = torch.stack([torch.randperm(D, generator=g)[:16] for _ in range(n_users)])
    sup_i = torch.stack([torch.randperm(D, generator=g)[:16] for _ in range(n_items)])
    UA.scatter_(1, sup_u, (torch.randint(0, 2, (n_users, 16), generator=g).float() * 2 - 1) / 4)
    IA.scatter_(1, sup_i, (torch.randint(0, 2, (n_items, 16), generator=g).float() * 2 - 1) / 4)
    users = torch.randperm(n_users, generator=g)[:B]
    items = torch.randperm(n_items, generator=g)[:2 * B]
    pos, neg = items[:B], items[B:]
    masks = []
    for q, sup in enumerate((sup_u[users], sup_u[users], sup_i[pos], sup_i[pos])):
        m = torch.rand(B, D, generator=g) < 0.8
        keep = sup if q % 2 == 0 else sup[:, :4]
        m.scatter_(1, sup, False)
        m.scatter_(1, keep, True)
        masks.append(m)
    return [t.to(dev) for t in (UA, IA, users, pos, neg)] + [[m.to(dev) for m in masks]]


@pytest.mark.parametrize("B", [1, 300, 20000])
@pytest.mark.parametrize("rw", [0.0, 0.1])
def test_op_equals_the_torch_expression_on_exact_inputs(dev, B, rw):
    UA, IA, users, pos, neg, masks = exact_operands(dev, B, seed=B)
    k = run_op(UA, IA, users, pos, neg, masks, 0.2, rw)
    t = run_torch(UA, IA, users, pos, neg, masks, 0.2, rw, k8=rw > 0)
    assert k[0].shape == t[0].shape == ()
    if B == 1:                                                         # no batch sum to order
        assert torch.equal(k[0], t[0])
    else:                                                              # the B log terms are summed in the kernel's order
        assert abs(k[0].item() - t[0].item()) <= 4 * U32 * (B + 8) * (abs(t[0].item()) + 1.0)
    if rw == 0:                                                        # unique rows: the scatter is a permutation
        assert torch.equal(k[1], t[1]) and torch.equal(k[2], t[2])
    else:
        for a, b in zip(k[1:], t[1:]):
            assert ((a - b).abs() <= 64 * U32 * b.abs() + 2 ** -12 * b.abs().max()).all()


def random_operands(dev, B, n_users, n_items, repeat, seed):
    g = torch.Generator().manual_seed(seed)
    UA, IA = torch.randn(n_users, 128, generator=g) * 0.1, torch.randn(n_items, 128, generator=g) * 0.1
    hi_u, hi_i = (5, 4) if repeat else (n_users, n_items)
    users = torch.randint(0, hi_u, (B,), generator=g)
    pos, neg = torch.randint(0, hi_i, (B,), generator=g), torch.randint(0, hi_i, (B,), generator=g)
    masks = [torch.rand(B, 128, generator=g) < 0.8 for _ in range(4)]
    return [t.to(dev) for t in (UA, IA, users, pos, neg)] + [[m.to(dev) for m in masks]]


@pytest.mark.parametrize("B,repeat", [(1, False), (2048, False), (2048, True), (20000, False)])
@pytest.mark.parametrize("rw", [0.0, 0.1])
def test_op_within_the_per_row_bound_of_float64(dev, B, repeat, rw):
    """The loss within 2^-16 of float64's (relative), each gradient row within 2^-12 of its largest float64 entry plus
    2^-20 of the table's: fp32 dots, norms and K8's 3xTF32 sums carry a few units of 2^-24 per step."""
    UA, IA, users, pos, neg, masks = random_operands(dev, B, 3000, 2000, repeat, seed=B)
    k = run_op(UA, IA, users, pos, neg, masks, 0.2, rw)
    t = run_torch(UA, IA, users, pos, neg, masks, 0.2, rw, dtype=torch.float64, k8=False)
    assert abs(k[0].item() - t[0].item()) <= 2 ** -16 * abs(t[0].item())
    for a, b in zip(k[1:], t[1:]):
        row = b.abs().amax(dim=1, keepdim=True)
        assert ((a.double() - b).abs() <= 2 ** -12 * row + 2 ** -20 * b.abs().max()).all()


@pytest.mark.parametrize("rw", [0.0, 0.1])
def test_zero_rows_follow_the_torch_expression(dev, rw):
    """A zero user row: its views' norms are 0, clamp_min's eps divides, and autograd's masked norm gradient is 0."""
    UA, IA, users, pos, neg, masks = exact_operands(dev, 64, seed=5)
    UA[users[3]] = 0.0
    IA[pos[7]] = 0.0
    k = run_op(UA, IA, users, pos, neg, masks, 0.2, rw)
    t = run_torch(UA, IA, users, pos, neg, masks, 0.2, rw, k8=rw > 0)
    assert abs(k[0].item() - t[0].item()) <= 4 * U32 * 72 * (abs(t[0].item()) + 1.0)
    for a, b in zip(k[1:], t[1:]):
        assert torch.isfinite(a).all()
        if rw == 0:
            assert torch.equal(a, b)
        else:
            assert ((a - b).abs() <= 64 * U32 * b.abs() + 2 ** -12 * b.abs().max()).all()


def test_nan_rows_follow_the_torch_expression(dev):
    """A NaN item row at reg_weight > 0: the loss is NaN, and so is every gradient entry the torch expression makes NaN
    (K8's sums over the NaN row reach every row)."""
    UA, IA, users, pos, neg, masks = exact_operands(dev, 64, seed=6)
    IA[pos[7]] = float("nan")
    k = run_op(UA, IA, users, pos, neg, masks, 0.2, 0.1)
    t = run_torch(UA, IA, users, pos, neg, masks, 0.2, 0.1)
    assert torch.isnan(k[0]) and torch.isnan(t[0])
    for a, b in zip(k[1:], t[1:]):
        assert torch.equal(torch.isnan(a), torch.isnan(b))


def test_op_gives_the_same_bits_on_every_run(dev):
    UA, IA, users, pos, neg, masks = random_operands(dev, 4000, 50, 30, True, seed=9)
    for rw in (0.0, 0.1):
        runs = [run_op(UA, IA, users, pos, neg, masks, 0.2, rw) for _ in range(2)]
        for a, b in zip(*runs):
            assert torch.equal(a, b)


@pytest.mark.parametrize("p", [0.2, 0.1, 0.3])
def test_dropout_scales_are_torchs(dev, p):
    """`native_dropout` on the device multiplies by `dropout_scales(p)[0]`, its backward by `[1]`."""
    from mmrec_b200 import ops
    x = (torch.randn(2048, 128, device=dev) * 0.1).requires_grad_(True)
    out, m = torch.native_dropout(x, p, True)
    g = torch.randn_like(out)
    out.backward(g)
    sf, sb = ops.dropout_scales(p)
    assert torch.equal(out, (x.detach() * m.float()) * sf)
    assert torch.equal(x.grad, (g * m.float()) * sb)


# ------------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------------
def make_env(shape):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_pgl_")
    u, i, e, d, f = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    if shape == "tiny":
        v, t = synth.make_features(i, f, seed=1)
    else:
        rng = np.random.default_rng(1)
        v, t = rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", gr, v, t)
    return os.path.join(tmp, "data") + "/"


@pytest.fixture(scope="module")
def env(dev):
    return make_env("tiny")


def recorded(model, gold, dev):
    """The recorded epoch's sub-graph and the recorded masks in place of the device draws."""
    model.sub_graph = model.pruner.adj_from_keep(torch.from_numpy(gold["keep_idx"]).to(dev))
    masks = [m.to(dev) for m in P.masks_of(gold)]
    model._dropout_masks = lambda *a: masks


def test_model_matches_reference(env, golden):
    from mmrec_b200.common.trainer import Trainer
    gold = golden("pgl_tiny.npz")
    config, train, valid, test, model = build("PGL", env, {})
    dev = config["device"]
    assert G.init_digests(model) == {k[len("init_sha256."):]: str(gold[k]) for k in gold.files if k.startswith("init_sha256.")}
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    recorded(model, gold, dev)
    model.eval()
    with torch.no_grad():
        for tag, adj in (("fwd_sub", model.sub_graph), ("fwd_norm", model.norm_adj)):
            for s, t in zip("ui", model.forward(adj)):
                assert G.rel(gold, f"{tag}_{s}", t.cpu().numpy()) < 1e-5, (tag, s)
    model.train()
    batch = torch.from_numpy(gold["batch"]).to(dev)
    named = dict(model.named_parameters())
    for p, rw in P.REG_CASES.items():
        model.reg_weight = rw
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(batch)
        loss.backward()
        assert tuple(loss.shape) == tuple(gold[p + "loss_shape"])
        np.testing.assert_allclose(loss.item(), gold[p + "loss"][0], rtol=1e-5)
        rec = [k[len(p + "grad."):] for k in G.recorded(gold, p + "grad.")]
        assert set(rec) == {k for k, q in named.items() if q.grad is not None}
        for k in rec:
            assert G.rel(gold, p + "grad." + k, named[k].grad.cpu().numpy()) < 1e-4, (p, k)
    model.zero_grad(set_to_none=True)
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_training_step_advances_the_device_generator_as_the_reference(env):
    """From one seed at dropout 0.2 and reg_weight 0.1: the device generator after `calculate_loss` equals its state after
    the reference's expressions (four nn.Dropout calls on [B, 2d]); the two losses agree within the op's bound."""
    config, train, valid, test, model = build("PGL", env, {})
    model.reg_weight = 0.1
    model.pre_epoch_processing()
    model.train()
    batch = next(iter(train)).to(config["device"])
    out = {}
    for route, fn in (("model", model.calculate_loss), ("reference", lambda b: P.reference_calculate_loss(model, b))):
        torch.cuda.manual_seed(77)
        with torch.no_grad():
            out[route] = (fn(batch).item(), torch.cuda.get_rng_state())
    assert torch.equal(out["model"][1], out["reference"][1])
    assert abs(out["model"][0] - out["reference"][0]) <= 2 ** -16 * abs(out["reference"][0])


def test_trajectory_through_fused_adam(env, golden):
    """Two epochs on the recorded batches with the recorded keep indices (dropout 0, reg_weight 0.1): every loss, the
    per-epoch metrics and the final state."""
    gold = golden("traj_pgl_tiny.npz")
    config, train, valid, test, model = build("PGL", env, dict(P.TRAJ_OVER))
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches, offs = gold["batches"], np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    b = 0
    for ep, nb in enumerate(gold["batches_per_epoch"]):
        model.sub_graph = model.pruner.adj_from_keep(torch.from_numpy(gold["keep_idx"][ep]).to(dev))
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
        assert G.rel(gold, "final." + k, q.cpu().numpy()) < 1e-4, k


def test_topk_equals_mask_topk_of_predict(env, golden):
    from mmrec_b200 import ops
    gold = golden("pgl_tiny.npz")
    config, train, valid, test, model = build("PGL", env, {})
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


@pytest.mark.parametrize("rw", [0.0, 0.1])
def test_training_step_replayed_from_a_cuda_graph_gives_the_eager_bits(env, golden, rw):
    """`calculate_loss` + `backward` (the recorded masks in place of the draws) captured once on a side stream and replayed:
    the loss and every gradient equal an eager step's bits."""
    gold = golden("pgl_tiny.npz")
    config, train, valid, test, model = build("PGL", env, {})
    dev = config["device"]
    recorded(model, gold, dev)
    model.reg_weight = rw
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


@pytest.mark.parametrize("rw", [0.0, 0.1])
def test_loss_at_clothing_shape_peaks_below_the_reference_expressions(dev, rw):
    """Peak memory of the loss after the tables, forward and backward, at clothing's shape (40 000 users, 23 000 items,
    2d = 128, B = 2048, dropout 0.2): the op with the model's four mask draws against the reference's expressions with its
    four nn.Dropout calls, which form the [B, B] similarity and exp matrices.  Each route is measured on its second call."""
    from mmrec_b200 import ops
    from mmrec_b200.utils import synth
    n_users, n_items = synth.SHAPES["clothing"][:2]
    g = torch.Generator(device=dev).manual_seed(3)
    UA = (torch.randn(n_users, 128, generator=g, device=dev) * 0.1).requires_grad_(True)
    IA = (torch.randn(n_items, 128, generator=g, device=dev) * 0.1).requires_grad_(True)
    B = 2048
    users = torch.randint(0, n_users, (B,), generator=g, device=dev)
    pos, neg = torch.randint(0, n_items, (B,), generator=g, device=dev), torch.randint(0, n_items, (B,), generator=g, device=dev)
    drop = torch.nn.Dropout(0.2)

    def ours():
        src = torch.empty(B, 128, device=dev)
        masks = [torch.native_dropout(src, 0.2, True)[1] for _ in range(4)]
        return ops.pgl_loss(UA, IA, users, pos, neg, masks, 0.2, rw)

    def reference():
        u, p, n = UA[users], IA[pos], IA[neg]
        mf = -torch.mean(torch.nn.functional.logsigmoid(torch.sum(u * p, dim=1) - torch.sum(u * n, dim=1)))
        cl = (P.info_nce(drop(u), drop(u)) + P.info_nce(drop(p), drop(p))) / 2
        return mf + rw * cl

    peaks = {}
    for name, fn in (("op", ours), ("reference", reference)):
        for _ in range(2):
            UA.grad = IA.grad = None
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn().backward()
            torch.cuda.synchronize()
            peaks[name] = torch.cuda.max_memory_allocated() - base
    UA.grad = IA.grad = None
    print(f"PGL loss at clothing's shape, reg_weight {rw}: peak {peaks['op'] / 2**20:.1f} MiB, reference expressions "
          f"{peaks['reference'] / 2**20:.1f} MiB")
    assert peaks["op"] < peaks["reference"]
