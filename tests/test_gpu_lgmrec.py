"""LGMRec on the device.  K8 (csrc/expsum.cu): `ops.expsum_rows` and its backward against fp64 within the bound derived in
the file's header, bit-reproducibility and the memory it takes at a quarter million rows.  The model class: golden
initial weights, forward, loss, gradients, scores, top-k and metrics recorded from the reference, with the reference's
Gumbel noise and dropout masks replayed."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _plan(nX, nY):
    """(chunks, Y tiles per chunk) of csrc/expsum.cu's es_plan."""
    xt, yt = -(-nX // 64), -(-nY // 64)
    if xt == 0 or yt == 0:
        return 0, 0
    c = min(-(-256 // xt), 32, yt)
    tpc = -(-yt // c)
    return -(-yt // tpc), tpc


def _eps_term(d, inv_tau, qt=1.0):
    """Relative error of one term e_bj (expsum.cu header), |q||t| <= qt."""
    delta = ((3 * d / 8 + 3) * 2 * U + 3 * 2.0 ** -22) * qt
    return delta * inv_tau + 2.0 ** -21


def _rows(n, d, seed, dup=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.nn.functional.normalize(torch.randn(n, d, generator=g, device="cuda"))
    if dup and n >= 8:
        x[5] = x[3]                                                   # users repeat in a batch
        x[7] = 0.0                                                    # a zero row (F.normalize keeps it zero)
    return x.contiguous()


def _check_kernel(B, M, d, seed=0):
    from mmrec_b200 import ops
    dev = _dev()
    tau, inv_tau = 0.2, 5.0
    q = _rows(B, d, seed)
    t = _rows(M, d, seed + 1)
    g = torch.rand(B, generator=torch.Generator(device="cuda").manual_seed(seed + 2), device=dev) * 2 - 1
    outs = []
    for _ in range(2):
        qq, tt = q.clone().requires_grad_(True), t.clone().requires_grad_(True)
        ttl = ops.expsum_rows(qq, tt, tau)
        ttl.backward(g)
        outs.append((ttl.detach(), qq.grad, tt.grad))
    for a, b in zip(outs[0], outs[1]):                                # bit-reproducible
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    ttl, dq, dt = outs[0]
    q64, t64, g64 = q.double(), t.double(), g.double()
    e = torch.exp((q64 @ t64.T) * inv_tau)                            # [B, M] in fp64
    ref = e.sum(1)
    eps = _eps_term(d, inv_tau, 1.0 + 1e-6)
    cq, tq = _plan(B, M)
    tol = 1.1 * (eps + (16 * tq + 2 + cq) * U)
    err = ((ttl.double() - ref).abs() / ref).max().item()
    assert err <= tol, f"ttl rel err {err:.3e} > bound {tol:.3e}"
    # backward, element-wise against the magnitude sums
    eps_b = eps + 3 * 2.0 ** -22 + 27 * 2 * U + 2 * U
    dq_ref = (g64 * inv_tau)[:, None] * (e @ t64)
    dq_mag = (g64.abs() * inv_tau)[:, None] * (e @ t64.abs())
    tol_q = 1.1 * (eps_b + (tq + cq) * U)
    err_q = ((dq.double() - dq_ref).abs() / dq_mag.clamp_min(1e-300)).max().item()
    assert err_q <= tol_q, f"dQ err {err_q:.3e} > bound {tol_q:.3e}"
    ct, tt_ = _plan(M, B)
    dt_ref = inv_tau * ((e * g64[:, None]).T @ q64)
    dt_mag = inv_tau * ((e * g64.abs()[:, None]).T @ q64.abs())
    tol_t = 1.1 * (eps_b + (tt_ + ct) * U)
    err_t = ((dt.double() - dt_ref).abs() / dt_mag.clamp_min(1e-300)).max().item()
    assert err_t <= tol_t, f"dT err {err_t:.3e} > bound {tol_t:.3e}"
    return err, err_q, err_t


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("B,M", [(2048, 7050), (2048, 19445), (2048, 40000), (1, 1), (77, 129)])
def test_expsum_rows_against_fp64(B, M, d):
    _check_kernel(B, M, d)


def test_expsum_rows_empty_tables():
    from mmrec_b200 import ops
    dev = _dev()
    q = _rows(33, 64, 0).requires_grad_(True)
    t = torch.empty(0, 64, device=dev, requires_grad=True)
    ttl = ops.expsum_rows(q, t, 0.2)
    assert torch.equal(ttl, torch.zeros(33, device=dev))
    ttl.sum().backward()
    assert torch.equal(q.grad, torch.zeros_like(q))
    q0 = torch.empty(0, 64, device=dev, requires_grad=True)
    t1 = _rows(100, 64, 1).requires_grad_(True)
    out = ops.expsum_rows(q0, t1, 0.2)
    assert out.shape == (0,)
    out.sum().backward()
    assert torch.equal(t1.grad, torch.zeros_like(t1))


def test_expsum_rows_overflow_matches_torch():
    """No maximum is subtracted, as in the reference: a row whose terms overflow gives inf, the others stay finite."""
    from mmrec_b200 import ops
    dev = _dev()
    q = _rows(70, 64, 3)
    t = _rows(300, 64, 4)
    q[10] = t[20] * 30.0                                              # <q, t> = 30 -> exp(150) overflows fp32
    got = ops.expsum_rows(q, t, 0.2)
    want = torch.exp(torch.matmul(q, t.T) / 0.2).sum(dim=1)
    assert torch.equal(torch.isinf(got), torch.isinf(want)) and bool(torch.isinf(got[10]))


def test_expsum_rows_memory_at_250k_rows():
    """B = 2048, M = 250 000, d = 64: forward + backward allocate the gradients and O((B + M) d) scratch; one [B, M] fp32
    matrix would be 2 GB."""
    from mmrec_b200 import ops
    dev = _dev()
    B, M, d = 2048, 250_000, 64
    q = _rows(B, d, 5).requires_grad_(True)
    t = _rows(M, d, 6).requires_grad_(True)
    g = torch.rand(B, device=dev)
    ops._ws_cache.clear()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    ttl = ops.expsum_rows(q, t, 0.2)
    ttl.backward(g)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    grads = q.grad.numel() * 4 + t.grad.numel() * 4
    assert peak - grads < 64 << 20, f"{(peak - grads) / 2**20:.1f} MiB besides the gradients"
    e = torch.exp((q[:64].detach().double() @ t.detach().double().T) * 5.0)
    c, tpc = _plan(B, M)
    tol = 1.1 * (_eps_term(d, 5.0, 1.0 + 1e-6) + (16 * tpc + 2 + c) * U)
    assert ((ttl[:64].detach().double() - e.sum(1)).abs() / e.sum(1)).max().item() <= tol


# ------------------------------------------------------------------------------------------------
# the model class against the reference (tests/golden/lgmrec_*.npz, traj_lgmrec_tiny.npz)
# ------------------------------------------------------------------------------------------------
import os  # noqa: E402
import sys  # noqa: E402

from test_gpu_models import build, check_topk, rel  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import lgmrec_golden  # noqa: E402

SETTINGS = {"lgmrec_tiny.npz": {}, "lgmrec_clothing_tiny.npz": {"n_hyper_layer": [2], "hyper_num": [64], "keep_rate": [0.2], "alpha": [0.2]}}


class Replay:
    """`F.gumbel_softmax` / `F.dropout` with the reference's CPU draws, in the order it made them (the device generator
    cannot reproduce that stream): Gumbel noise g -> softmax((logits + g) / tau), scaled mask m -> input * m."""

    def __init__(self, draws, device):
        self.draws, self.device = list(draws), device
        self._saved = None

    def _next(self, shape):
        a = self.draws.pop(0)
        assert tuple(a.shape) == tuple(shape), f"draw of shape {a.shape} where {tuple(shape)} is drawn"
        return torch.from_numpy(a).to(self.device)

    def gumbel_softmax(self, logits, tau=1.0, hard=False, eps=1e-10, dim=-1):
        return ((logits + self._next(logits.shape)) / tau).softmax(dim)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        if not training or p == 0 or input.numel() == 0:
            return input
        return input * self._next(input.shape)

    def __enter__(self):
        import torch.nn.functional as F
        self._saved = (F.gumbel_softmax, F.dropout)
        F.gumbel_softmax, F.dropout = self.gumbel_softmax, self.dropout
        return self

    def __exit__(self, *exc):
        import torch.nn.functional as F
        F.gumbel_softmax, F.dropout = self._saved


def _draws(gold, prefix):
    """The trajectory's recorded draws, in order."""
    return [gold["%sdraw%d" % (prefix, k)] for k in range(int(gold[prefix + "n_draws"]))]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import os
    import tempfile
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_")
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, v, t)
    return os.path.join(tmp, "data") + "/"


@pytest.mark.parametrize("gfile", list(SETTINGS))
def test_lgmrec_matches_reference(env, gfile):
    gold = lgmrec_golden.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", gfile))
    config, train, valid, test, model = build("LGMRec", env, SETTINGS[gfile])
    dev = config["device"]
    for k, p in model.state_dict().items():
        assert np.array_equal(p.cpu().numpy(), gold["param0." + k]), f"initial {k} differs from the reference"
    assert [k for k, _ in model.named_parameters()] == list(gold["param_order"])
    assert np.array_equal(model.num_inters.cpu().numpy(), gold["num_inters"])
    model.eval()
    with Replay(lgmrec_golden.regenerate(gold, "fwd_"), dev) as r, torch.no_grad():
        u, i, hyp = model.forward()
    assert not r.draws
    assert rel(u, gold["fwd_u"]) < 1e-5 and rel(i, gold["fwd_i"]) < 1e-5
    for n, h in zip(("uv", "iv", "ut", "it"), hyp):
        assert rel(h, gold["fwd_hyper_" + n]) < 1e-5, n
    model.train()
    model.zero_grad()
    with Replay(lgmrec_golden.regenerate(gold, "loss_"), dev) as r:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    assert not r.draws
    loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy().reshape(-1), gold["loss"], rtol=2e-5)
    named = dict(model.named_parameters())
    ref_grads = {k[5:]: gold[k] for k in gold.files if k.startswith("grad.")}
    assert set(ref_grads) == {k for k, p in named.items() if p.requires_grad}
    gmax = max(float(np.abs(g).max()) for g in ref_grads.values())
    for k, gref in ref_grads.items():
        err = (named[k].grad.detach().cpu().double() - torch.from_numpy(gref).double()).norm().item()
        assert err < 1e-4 * float(np.linalg.norm(gref)) + 1e-7 * gmax * np.sqrt(gref.size), f"grad {k}"
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    scale = float(np.abs(gold["scores"]).max())
    with torch.no_grad():
        with Replay(lgmrec_golden.regenerate(gold, "scores_"), dev):
            scores = model.full_sort_predict(eb)
        assert (scores.cpu() - torch.from_numpy(gold["scores"])).abs().max().item() < 2e-5 * scale
        with Replay(lgmrec_golden.regenerate(gold, "scores_"), dev):                  # the fused route runs its own forward on the same draws
            idx = model.full_sort_topk(eb, 50)
        check_topk(idx, gold["scores"], gold["eval_mask"], 50, scale)
    from mmrec_b200.common.trainer import Trainer
    tr = Trainer(config, model)
    with Replay(lgmrec_golden.regenerate(gold, "valid_"), dev) as r:
        res = tr.evaluate(valid)
    assert not r.draws
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    with Replay(lgmrec_golden.regenerate(gold, "test_"), dev) as r:
        res_t = tr.evaluate(test, is_test=True)
    assert not r.draws
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_lgmrec_trajectory_replay(env, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches and draws: per-batch losses, per-epoch metrics."""
    gold = golden("traj_lgmrec_tiny.npz")
    config, train, valid, test, model = build("LGMRec", env, {})
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches = torch.from_numpy(gold["batches"])
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    b = 0
    with Replay(_draws(gold, ""), dev) as r:
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
