"""DRAGON on the GPU: the model class against the golden files recorded from the reference
(tests/golden/make_golden_dragon.py): initial state, `mm_adj`, the sample, the mutated batch, `user_rep`, `result_embed`,
the loss, every gradient, the scores, the top-50 and the metrics, for both modalities, text only and 'mean'; two epochs
through FusedAdam; one training step replayed from a CUDA graph gives the eager bits."""
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
from make_golden_dragon import CASES  # noqa: E402
from test_gpu_models import build  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


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
def envs(dev):
    return {False: _env(False), True: _env(True)}


def _sub(gold, p):
    return {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)} if p else {k: gold[k] for k in gold.files}


def _overrides(p):
    return {k: [v] for k, v in CASES[p][0].items()}


def _user_rep(model):
    U = model.n_users
    if model.v_rep is not None and model.t_rep is not None:
        w = model.weight_u.detach()
        return torch.cat((model.v_rep[:U, :, 0] * w[:, 0], model.t_rep[:U, :, 0] * w[:, 1]), dim=1).detach()
    return (model.t_rep if model.t_rep is not None else model.v_rep)[:U].detach()


@pytest.mark.parametrize("p", list(CASES))
def test_dragon_matches_reference(envs, golden, p):
    from mmrec_b200.common.trainer import Trainer
    gold = _sub(golden("dragon_tiny.npz"), p)
    config, train, valid, test, model = build("DRAGON", envs[CASES[p][1]], _overrides(p))
    dev = config["device"]
    init = {k[len("init_sha256."):]: str(v) for k, v in gold.items() if k.startswith("init_sha256.")}
    assert G.init_digests(model) == init, "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    assert "result_embed" not in dict(model.named_parameters())
    assert G.sha256_tagged(model.result_embed.cpu().numpy()) == str(gold["result_embed0_sha256"])
    n_i = model.n_items
    mm = torch.zeros(n_i, n_i, dtype=torch.float64)
    mm[tuple(torch.from_numpy(gold["mm_adj_indices"]))] = torch.from_numpy(gold["mm_adj_values"]).double()
    r, c, v = model.mm_adj.coo()
    got = torch.zeros(n_i, n_i, dtype=torch.float64).index_put_((r.cpu(), c.cpu()), v.cpu().double(), accumulate=True)
    assert torch.equal(got != 0, mm != 0) and (got - mm).abs().max().item() <= 1e-6 * mm.abs().max().item()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    model.eval()
    with torch.no_grad():
        s0 = model.full_sort_predict(eb)
        assert s0.dtype == torch.float64 and s0.is_cuda
        rows = gold["scores0_rows"]
        np.testing.assert_allclose(s0[:len(rows)].cpu().numpy(), rows, rtol=1e-12, atol=1e-13)
        idx0 = model.full_sort_topk(eb, 50)
        m = s0.clone()
        m[eb[1][0], eb[1][1]] = -1e10
        assert torch.equal(idx0, torch.topk(m, 50, dim=-1)[1])
    np.random.seed(D.SAMPLE_SEED)
    model.pre_epoch_processing()
    assert G.equal(gold, "sample_idx", model.epoch_user_graph.numpy())
    assert G.equal(gold, "sample_w", model.user_weight_matrix.cpu().numpy())
    model.train()
    model.zero_grad()
    b = torch.from_numpy(gold["batch"]).to(dev)
    loss = model.calculate_loss(b)
    assert np.array_equal(b.cpu().numpy(), gold["batch_after"])       # the reference's in-place item offset
    assert G.rel(gold, "user_rep", _user_rep(model).cpu().numpy()) < 1e-5
    assert G.rel(gold, "result_embed", model.result_embed.detach().cpu().numpy()) < 1e-5
    assert model.result_embed.dtype == torch.float32 and model.result_embed.shape[1] == (64 if CASES[p][1] else 128)
    assert isinstance(model.t_preference, torch.nn.Parameter) and "t_preference" in dict(model.named_parameters())
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
        assert G.rel(gold, "scores", s.cpu().numpy()) < 1e-5
        idx = model.full_sort_topk(eb, 50).cpu()
        want = torch.from_numpy(gold["topk50"])
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10
        m = m.cpu().double()
        scale = m[m > -1e9].abs().max().item()
        diff = idx != want                                              # every difference is a near tie of the scores
        gap = (m.gather(1, idx) - m.gather(1, want)).abs()
        assert (gap[diff] <= 1e-5 * scale).all() and diff.float().mean().item() < 0.05
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_dragon_trajectory_replay(envs, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches, `np.random` seeded before each epoch's sample:
    per-batch losses and per-epoch metrics."""
    gold = golden("traj_dragon_tiny.npz")
    config, train, valid, test, model = build("DRAGON", envs[False], {})
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


def test_training_step_replayed_from_a_cuda_graph_gives_the_eager_bits(envs, golden):
    """`calculate_loss` + `backward` captured once on a side stream and replayed: the loss, `result_embed` and every
    gradient equal an eager step's bits on the same batch (the batch is restored before each run: the forward offsets its
    item columns in place)."""
    gold = golden("dragon_tiny.npz")
    config, train, valid, test, model = build("DRAGON", envs[False], {})
    dev = config["device"]
    np.random.seed(D.SAMPLE_SEED)
    model.pre_epoch_processing()
    model.train()
    batch0 = torch.from_numpy(gold["batch"]).to(dev)
    static = batch0.clone()
    params = [q for q in model.parameters() if q.requires_grad]

    def step():
        loss = model.calculate_loss(static)
        loss.backward()
        return loss

    def snapshot(loss):
        return [loss.detach().clone(), model.result_embed.detach().clone()] + \
               [q.grad.clone() if q.grad is not None else None for q in params]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            static.copy_(batch0)
            model.zero_grad(set_to_none=True)
            step()
    torch.cuda.synchronize()
    static.copy_(batch0)
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        loss_c = step()
    torch.cuda.synchronize()
    runs = []
    for _ in range(2):
        static.copy_(batch0)
        for q in params:
            if q.grad is not None:
                q.grad.zero_()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            g.replay()
        torch.cuda.synchronize()
        runs.append(snapshot(loss_c))
    grads_c = [q.grad for q in params]
    for q in params:                                                     # the eager step, outside the graph's memory
        q.grad = None
    static.copy_(batch0)
    with torch.cuda.stream(side):
        eager = snapshot(step())
    torch.cuda.synchronize()
    for run in runs:
        assert len(run) == len(eager)
        for a, e in zip(run, eager):
            assert (a is None) == (e is None)
            if a is not None:
                assert torch.equal(a, e)
    assert any(q is not None for q in grads_c)
