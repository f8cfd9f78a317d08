"""MVGAE on the device.  `ops.max_dot` (K3's fused score + top-1 with a gather / `index_sum_rows` backward): bit for bit
against `score_topk(k = 1)` and the exact fp32 top-k oracle, the argmax against an fp64 re-score, ties, NaN, gradients
against torch's autograd of the reference's [B, B, d] expression, run-to-run bit equality and its memory at B = 8192.  The
model class: golden initial weights, forward, decodes, loss, gradients, scores, top-k and metrics recorded from the
reference, with the reference's dropout masks and Gaussian noise replayed, and two epochs through FusedAdam."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _gamma(d):
    u = 2.0 ** -24
    return d * u / (1 - d * u)


def _ref_expr(z, user, neg_items):
    """`dot_product_decode_neg` without the sigmoid (src/models/mvgae.py:76-84): the [B, B, d] product."""
    users = torch.unsqueeze(user, 1)
    re_users = users.repeat(1, neg_items.size(0))
    neg_values = torch.sum(z[re_users] * z[neg_items], -1)
    return torch.max(neg_values, dim=-1)


def _check_near_ties(q, t, got_idx, want_idx):
    """Rows whose argmax differs must be near ties: fp64 scores within the fp32 bound 2 gamma_d sum_k |q_k t_k|."""
    q64, t64 = q.double(), t.double()
    bad = torch.nonzero(got_idx != want_idx).flatten()
    for b in bad.tolist():
        i, j = int(got_idx[b]), int(want_idx[b])
        gap = abs(float(q64[b] @ t64[i]) - float(q64[b] @ t64[j]))
        bound = 2 * _gamma(q.shape[1]) * max(float(q64[b].abs() @ t64[i].abs()), float(q64[b].abs() @ t64[j].abs()))
        assert gap <= bound, f"row {b}: argmax {i} vs {j}, gap {gap} beyond the fp32 bound {bound}"
    return bad.numel()


@pytest.mark.parametrize("B,M,d,sig", [(64, 100, 64, True), (2048, 2048, 64, True), (1000, 5000, 32, False), (700, 3000, 128, False)])
def test_max_dot_is_score_topk_k1(B, M, d, sig):
    from mmrec_b200 import ops
    from oracle import mmrec_oracle as O
    dev = _dev()
    g = torch.Generator(device="cuda").manual_seed(B + M + d)
    q = torch.randn(B, d, generator=g, device=dev)
    t = torch.randn(M, d, generator=g, device=dev)
    if sig:                                                           # MVGAE's operands: sigmoid(z), all scores positive and close
        q, t = torch.sigmoid(q), torch.sigmoid(t)
    t[7] = t[3]                                                       # a duplicate row
    v, i = ops.max_dot(q, t)
    assert v.shape == (B,) and i.shape == (B,) and i.dtype == torch.int64 and v.dtype == torch.float32
    sv, si = ops.score_topk(q, t, None, None, 1)
    assert torch.equal(v, sv[:, 0]) and torch.equal(i, si[:, 0])
    rv, ri = O.cf_exact_topk(q, t, None, None, 1, device=dev)
    assert torch.equal(v.cpu(), rv[:, 0]) and torch.equal(i.cpu(), ri[:, 0])
    s64 = q.double() @ t.double().T
    _check_near_ties(q, t, i, s64.argmax(dim=1))
    assert (v.double() - s64.max(dim=1).values).abs().max().item() <= 2 * _gamma(d) * float((q.abs().double() @ t.abs().double().T).max())


def test_max_dot_ties_take_the_lowest_index():
    from mmrec_b200 import ops
    dev = _dev()
    d = 64
    q = torch.ones(3, d, device=dev)
    t = torch.zeros(10, d, device=dev)
    t[:, 0] = torch.arange(10, dtype=torch.float32, device=dev) * 0.125          # all below 3
    t[2, :2] = torch.tensor([1.0, 2.0])                                # distinct rows, same exact score 3
    t[5, :2] = torch.tensor([2.0, 1.0])
    t[8, :3] = torch.tensor([0.5, 0.5, 2.0])
    v, i = ops.max_dot(q, t)
    assert torch.equal(i.cpu(), torch.full((3,), 2)) and torch.equal(v.cpu(), torch.full((3,), 3.0))
    t2 = t.clone()
    t2[1] = t2[9] = torch.full((d,), 0.25, device=dev)                  # duplicates, both the max (score 16)
    v, i = ops.max_dot(q, t2)
    assert torch.equal(i.cpu(), torch.full((3,), 1)) and torch.equal(v.cpu(), torch.full((3,), 16.0))
    q0 = torch.zeros(2, d, device=dev)                                 # every score +0: the first column
    v, i = ops.max_dot(q0, t)
    assert torch.equal(i.cpu(), torch.zeros(2, dtype=torch.int64)) and torch.equal(v.cpu(), torch.zeros(2))


def test_max_dot_nan_is_the_max_at_its_first_column():
    """As `torch.max`: a row with a NaN score returns NaN at its first NaN column -- whichever NaN went in (the device's
    sigmoid of a NaN, or a negative NaN bit pattern)."""
    from mmrec_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(6, 64, generator=g, device=dev)
    y = torch.randn(40, 64, generator=g, device=dev)
    neg_nan = -4194304                                                 # int32 bits 0xFFC00000: a NaN with the sign bit set
    y[11, 3] = float("nan")
    y.view(torch.int32)[25, 0] = neg_nan
    x[4, 9] = float("nan")
    q, t = torch.sigmoid(x), torch.sigmoid(y)                          # the device's sigmoid of a NaN
    t.view(torch.int32)[30, 1] = neg_nan                               # and a negative NaN as it is
    assert torch.isnan(t[30, 1]) and t.view(torch.int32)[30, 1].item() < 0
    v, i = ops.max_dot(q, t)
    want_v, want_i = torch.max(torch.sum(q.cpu()[:, None, :] * t.cpu()[None, :, :], -1), dim=-1)
    assert torch.isnan(v).all() and torch.isnan(want_v).all()
    assert torch.equal(i.cpu(), want_i)
    assert i.tolist() == [11, 11, 11, 11, 0, 11]
    q2 = torch.sigmoid(x)
    q2[4] = torch.sigmoid(x[3])                                         # no NaN in q: the first NaN column of t
    v, i = ops.max_dot(q2, t[20:])
    assert torch.isnan(v).all() and i.tolist() == [5] * 6


@pytest.mark.parametrize("B", [256, 1024])
def test_max_dot_gradients_against_the_reference_expression(B):
    """z, users and negatives as MVGAE's decode sees them (ids repeat: repeated argmax targets); the loss weights each
    row's max.  Gradients of z through our op and through torch's autograd of the [B, B, d] expression."""
    from mmrec_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cuda").manual_seed(B)
    N, d = 3 * B // 2, 64
    z0 = torch.randn(N, d, generator=g, device=dev)
    user = torch.randint(0, N, (B,), generator=g, device=dev)
    neg = torch.randint(0, N, (B,), generator=g, device=dev)
    w = torch.randn(B, generator=g, device=dev)
    z = z0.clone().requires_grad_(True)
    v, i = ops.max_dot(z[user], z[neg])
    (w * v).sum().backward()
    gz = z.grad.clone()
    zr = z0.clone().requires_grad_(True)
    rv, ri = _ref_expr(zr, user, neg)
    (w * rv).sum().backward()
    assert _check_near_ties(z0[user], z0[neg], i, ri) == 0             # (these seeds: no near tie, so the gradients compare)
    assert (v - rv).abs().max().item() <= 2 * _gamma(d) * float((z0[user].abs() @ z0[neg].abs().T).max())
    gref = zr.grad.double()
    err = (gz.double() - gref).norm().item()
    assert err < 1e-4 * gref.norm().item() + 1e-7 * gref.abs().max().item() * np.sqrt(gref.numel())
    # run to run: bit-identical values, indices and gradients (many rows share an argmax target)
    assert torch.bincount(i).max().item() > 1
    for _ in range(2):
        z2 = z0.clone().requires_grad_(True)
        v2, i2 = ops.max_dot(z2[user], z2[neg])
        (w * v2).sum().backward()
        assert torch.equal(v2, v) and torch.equal(i2, i) and torch.equal(z2.grad, gz)


def test_max_dot_gradient_of_each_operand():
    """dq = g t[index], dt = sum over the rows that selected j of g q, in ascending b (bitwise: `index_sum_rows`)."""
    from mmrec_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(500, 64, generator=g, device=dev).requires_grad_(True)
    t = torch.randn(40, 64, generator=g, device=dev).requires_grad_(True)
    w = torch.randn(500, generator=g, device=dev)
    v, i = ops.max_dot(q, t)
    dq, dt = torch.autograd.grad((w * v).sum(), (q, t))
    assert torch.equal(dq, w[:, None] * t.detach()[i])
    want = torch.zeros_like(t)
    for b in range(500):                                               # ascending b, one fp32 add at a time
        want[i[b]] += w[b] * q.detach()[b]
    assert torch.equal(dt, want)
    assert ops.max_dot(q, t)[1].requires_grad is False


def test_max_dot_memory_at_8192():
    """Forward + backward at B = M = 8192, d = 64 take O(B d) beyond the inputs and their gradients (the reference's
    expression would build a 16 GiB [B, B, d] tensor, and its backward another; it is not run here)."""
    from mmrec_b200 import ops
    dev = _dev()
    B, d = 8192, 64
    g = torch.Generator(device="cuda").manual_seed(8)
    q = torch.sigmoid(torch.randn(B, d, generator=g, device=dev)).requires_grad_(True)
    t = torch.sigmoid(torch.randn(B, d, generator=g, device=dev)).requires_grad_(True)
    w = torch.randn(B, generator=g, device=dev)
    torch.autograd.grad((w * ops.max_dot(q, t)[0]).sum(), (q, t))     # sizes the score_topk workspace (kept across calls)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    v, i = ops.max_dot(q, t)
    dq, dt = torch.autograd.grad((w * v).sum(), (q, t))
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - dq.numel() * 4 - dt.numel() * 4
    assert extra < 4 << 20, f"{extra / 2 ** 20:.1f} MiB beyond the inputs and gradients"
    from mmrec_b200 import _lib
    assert _lib.load().mmrec_score_topk_workspace_bytes(B, B, d, 1) < 80 << 20      # the cached K3 scratch stays bounded


# ------------------------------------------------------------------------------------------------
# the model class against the reference's golden files
# ------------------------------------------------------------------------------------------------
sys.path.insert(0, os.path.join(HERE, "golden"))
import golden_io as G  # noqa: E402
import mvgae_golden  # noqa: E402
from test_gpu_models import build, check_topk, rel  # noqa: E402


class Replay:
    """`F.dropout` / `torch.randn_like` with the reference's CPU draws, in the order it made them (the device generator
    cannot reproduce that stream): scaled mask m -> input * m, Gaussian noise -> the recorded tensor."""

    def __init__(self, draws, device):
        self.draws, self.device = list(draws), device
        self._saved = None

    def _next(self, shape):
        a = self.draws.pop(0)
        assert tuple(a.shape) == tuple(shape), f"draw of shape {a.shape} where {tuple(shape)} is drawn"
        return torch.from_numpy(a).to(self.device)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        if not training or p == 0 or input.numel() == 0:
            return input
        return input * self._next(input.shape)

    def randn_like(self, input, **kw):
        return self._next(input.shape)

    def __enter__(self):
        import torch.nn.functional as F
        self._saved = (F.dropout, torch.randn_like)
        F.dropout, torch.randn_like = self.dropout, self.randn_like
        return self

    def __exit__(self, *exc):
        import torch.nn.functional as F
        F.dropout, torch.randn_like = self._saved


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


def test_mvgae_matches_reference(env, golden, monkeypatch):
    from mmrec_b200 import ops
    gold = golden("mvgae_tiny.npz")
    config, train, valid, test, model = build("MVGAE", env, {})
    dev = config["device"]
    assert G.same_init(model, gold, mvgae_golden.plain(model)) == [], "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == list(gold["param_order"])
    model.eval()
    with Replay([], dev), torch.no_grad():
        fwd = model.forward()
    assert rel(fwd[0], gold["fwd_pd_mu"]) < 1e-5
    assert torch.equal(fwd[2], fwd[0])                                  # evaluation mode: z is pd_mu
    decodes = []
    real = ops.max_dot

    def spy(q, t):
        v, i = real(q, t)
        decodes.append((q.detach(), t.detach(), v.detach(), i))
        return v, i
    monkeypatch.setattr(ops, "max_dot", spy)
    model.train()
    model.zero_grad()
    with Replay(mvgae_golden.regenerate(gold, "loss_"), dev) as r:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    assert not r.draws
    loss.backward()
    monkeypatch.setattr(ops, "max_dot", real)
    np.testing.assert_allclose(loss.detach().cpu().numpy().reshape(-1), gold["loss"], rtol=2e-6)
    assert len(decodes) == 4
    for c, (q, t, v, i) in enumerate(decodes):
        assert rel(v, gold["decode_val"][c]) < 1e-6
        _check_near_ties(q, t, i, torch.from_numpy(gold["decode_arg"][c]).to(dev))
    named = dict(model.named_parameters())
    ref_grads = {k[5:]: gold[k] for k in gold.files if k.startswith("grad.")}
    assert set(ref_grads) == {k for k, p in named.items() if p.grad is not None}
    gmax = max(float(np.abs(g).max()) for g in ref_grads.values())
    for k, gref in ref_grads.items():
        err = (named[k].grad.detach().cpu().double() - torch.from_numpy(gref).double()).norm().item()
        assert err < 1e-4 * float(np.linalg.norm(gref)) + 1e-7 * gmax * np.sqrt(gref.size), f"grad {k}"
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    scale = float(np.abs(gold["scores"]).max())
    with torch.no_grad():
        scores = model.full_sort_predict(eb)
        assert (scores.cpu() - torch.from_numpy(gold["scores"])).abs().max().item() < 2e-5 * scale
        check_topk(model.full_sort_topk(eb, 50), gold["scores"], gold["eval_mask"], 50, scale)
    from mmrec_b200.common.trainer import Trainer
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_mvgae_trajectory_replay(env, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches and draws: per-batch losses, per-epoch metrics
    (scored from the last training forward's `result_embed`)."""
    gold = golden("traj_mvgae_tiny.npz")
    config, train, valid, test, model = build("MVGAE", env, {})
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches = torch.from_numpy(gold["batches"])
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    b = 0
    with Replay(mvgae_golden.trajectory_draws(gold), dev) as r:
        for ep, nb in enumerate(gold["batches_per_epoch"]):
            model.pre_epoch_processing()
            model.train()
            for _ in range(int(nb)):
                trainer.optimizer.zero_grad()
                loss = model.calculate_loss(batches[:, offs[b]:offs[b + 1]].to(dev))
                np.testing.assert_allclose(loss.item(), gold["losses"][b], rtol=5e-5)
                loss.backward()
                trainer.optimizer.step()
                b += 1
            trainer.lr_scheduler.step()
            v = trainer.evaluate(valid)
            t = trainer.evaluate(test, is_test=True)
            np.testing.assert_allclose([v[k] for k in names], gold["valid"][ep], atol=2e-4)
            np.testing.assert_allclose([t[k] for k in names], gold["test"][ep], atol=2e-4)
    assert not r.draws
