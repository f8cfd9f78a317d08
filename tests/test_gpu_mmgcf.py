"""MMGCF on the GPU: the late-fusion kernel (`ops.late_fuse`, csrc/fuse.cu) against the reference's torch expression run
on the device, and the model class against the golden files recorded from the reference (tests/golden/make_golden_mmgcf.py).

- Forward, equal / alpha: `torch.equal` with the torch expression on the device (NaN in the same places), every
  element-wise mode, one and two modalities, d = 32 / 64 / 128, idx absent, repeated and unsorted, n = 1 and n past two
  sweeps of the grid, zero and NaN rows.  This pins the rounding the kernel follows: a mean of three terms is the sum times
  fl(1/3) on the device (the CPU divides by 3).
- Forward, normalized: within 8 fp32 ulps of the row scale (the row norm is a reduction in another order), all-zero rows
  (the 1e-12 clamp) exactly 0.
- Backward: equal / alpha bit for bit with autograd of the expression (d alpha to fp32 reorder error, and the same bits on
  every run); normalized within the bound.
- Model: all cases of the golden files; the two-epoch trajectories through FusedAdam with the recorded pruning draws;
  `full_sort_topk` against `mask_topk` of `full_sort_predict`; the gathered training route against the reference's
  full-table expressions on the device."""
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
import mmgcf_golden as M  # noqa: E402
from test_gpu_models import build  # noqa: E402

MODES = [(f, w) for f in ("mean", "sum") for w in ("equal", "alpha", "normalized")]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def same(a, b):
    """Equal values, NaN where the other has NaN (torch.equal alone is False on NaN)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0), b.masked_fill(nb, 0))


def _operands(dev, n_items, n, d, mods, idx_kind, seed=0, special=True):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    E = torch.randn(n_items, d, generator=gen)
    if idx_kind is None:
        idx, n = None, n_items
    elif idx_kind == "repeat":
        idx = torch.randint(0, n_items, (n,), generator=gen)
        idx[: n // 2] = idx[n // 2: 2 * (n // 2)]
    else:
        idx = torch.randperm(n_items, generator=gen)[:n]
    feats = [torch.randn(n, d, generator=gen) * 3 for _ in range(mods)]
    if special and n >= 4:
        E[(idx[0] if idx is not None else 0)] = 0                      # a zero row of each table
        feats[0][1] = 0
        feats[-1][2] = float("nan")
        E[(idx[3] if idx is not None else 3), 5] = float("nan")
    alpha = torch.sigmoid(torch.randn((), generator=gen)).reshape(1)
    to = lambda x: None if x is None else x.to(dev)
    return to(E), [to(f) for f in feats], to(idx), to(alpha)


CASES = [(d, mods, idx_kind, n_items, n) for d in (32, 64, 128) for mods in (1, 2)
         for idx_kind, n_items, n in ((None, 300, None), ("repeat", 50, 97), ("perm", 400, 300))] + \
        [(64, 2, None, 1, None), (64, 2, "repeat", 7, 1), (128, 2, None, 2 * 8 * 8 * 132 + 37, None)]


@pytest.mark.parametrize("fusion,weighting", MODES)
@pytest.mark.parametrize("d,mods,idx_kind,n_items,n", CASES)
def test_forward_and_backward_against_the_torch_expression(dev, fusion, weighting, d, mods, idx_kind, n_items, n):
    from mmrec_b200 import ops
    E, feats, idx, alpha = _operands(dev, n_items, n, d, mods, idx_kind)
    al = alpha if weighting == "alpha" else None
    v, t = (feats[0], feats[1]) if mods == 2 else (None, feats[0])
    got = ops.late_fuse(E, v, t, fusion, weighting, alpha=al, idx=idx)
    want = M.torch_late_fuse(E, v, t, fusion, weighting, alpha=al, idx=idx)
    if weighting != "normalized":
        assert same(got, want)
    else:
        fin = torch.isfinite(want)
        assert torch.equal(fin, torch.isfinite(got))
        scale = want.abs().masked_fill(~fin, 0).amax(dim=1, keepdim=True).clamp_min(1e-30)
        assert ((got - want).abs().masked_fill(~fin, 0) <= 8 * 2.0 ** -24 * scale).all()

    # backward on finite operands (NaN gradients only spread NaN)
    E, feats, idx, alpha = _operands(dev, n_items, n, d, mods, idx_kind, seed=1, special=False)
    ins = [E] + feats + ([alpha] if weighting == "alpha" else [])
    outs = []
    g = torch.randn(got.shape, generator=torch.Generator(device="cpu").manual_seed(2)).to(dev)
    for fn in (ops.late_fuse, M.torch_late_fuse):
        xs = [x.clone().requires_grad_() for x in ins]
        vv, tt = (xs[1], xs[2]) if mods == 2 else (None, xs[1])
        y = fn(xs[0], vv, tt, fusion, weighting, alpha=xs[-1] if weighting == "alpha" else None, idx=idx)
        y.backward(g)
        outs.append([x.grad for x in xs])
    for k, (a, b) in enumerate(zip(*outs)):
        if weighting == "alpha" and k == len(ins) - 1:                   # a sum over every element: reorder error
            mag = (g.abs() * ((E if idx is None else E[idx]).abs() + sum(f.abs() for f in feats))).sum().item()
            assert abs(a.item() - b.item()) <= 1e-5 * mag, (a, b)
        elif weighting == "normalized":
            assert ((a - b).abs() <= 1e-5 * b.abs().amax(dim=1, keepdim=True).clamp_min(1e-30)).all(), k
        elif k == 0 and idx is not None and idx_kind == "repeat":
            assert ((a - b).abs() <= 1e-6 * b.abs().max()).all()            # autograd's index backward adds in its own order
        else:
            assert torch.equal(a, b), k


@pytest.mark.parametrize("fusion", ["mean", "sum"])
def test_dalpha_is_the_same_bits_on_every_run(dev, fusion):
    from mmrec_b200 import ops
    E, feats, idx, alpha = _operands(dev, 5000, 8000, 64, 2, "repeat", special=False)
    g = torch.randn(8000, 64, device=dev)
    res = []
    for _ in range(3):
        a = alpha.clone().requires_grad_()
        ops.late_fuse(E, feats[0], feats[1], fusion, "alpha", alpha=a, idx=idx).backward(g)
        res.append(a.grad.clone())
    assert all(torch.equal(res[0], r) for r in res[1:])


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
    return os.path.join(tmp, "data") + "/"


@pytest.fixture(scope="module")
def envs(dev):
    return {False: _env(False), True: _env(True)}


@pytest.mark.parametrize("name", list(M.CASES))
def test_mmgcf_matches_reference(envs, golden, name):
    from mmrec_b200.common.trainer import Trainer
    gold = golden("mmgcf_tiny.npz")
    fusion, weighting, layers, text_only = M.CASES[name]
    sub = {k[len(name) + 1:]: gold[k] for k in gold.files if k.startswith(name + ".")}
    config, train, valid, test, model = build("MMGCF", envs[text_only], M.overrides(fusion, weighting, layers))
    dev = config["device"]
    init = {k[len("init_sha256."):]: str(v) for k, v in sub.items() if k.startswith("init_sha256.")}
    assert G.init_digests(model) == init, "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]
    assert G.equal(gold, "edge_values", model.edge_values.cpu().numpy())
    model.masked_adj = model.pruner.adj_from_keep(torch.from_numpy(gold["prune_keep_idx"]).to(dev))
    model.eval()
    with torch.no_grad():
        u, i = model.forward(model.norm_adj)
        _, im = model.forward(model.masked_adj)
    assert G.rel(sub, "fwd_i", i.cpu().numpy()) < 1e-5 and G.rel(sub, "fwd_masked_i", im.cpu().numpy()) < 1e-5
    if "fwd_u.sha256" in sub:
        assert G.rel(sub, "fwd_u", u.cpu().numpy()) < 1e-5
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    loss.backward()
    np.testing.assert_allclose(loss.item(), sub["loss"][0], rtol=1e-5)
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(sub, "grad.")]
    assert set(grads) == {k for k, q in named.items() if q.grad is not None}
    err = M.grad_errors(sub, {k: named[k].grad.cpu().numpy() for k in grads})
    assert max(err.values()) < 2e-4, err
    model.zero_grad()
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        assert G.rel(sub, "scores", model.full_sort_predict(eb).cpu().numpy()) < 1e-5
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in sub["metric_names"]]), sub["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in sub["metric_names"]]), sub["test_metric_values"], atol=1e-4 + 1e-12)


@pytest.mark.parametrize("name", list(M.TRAJ))
def test_mmgcf_trajectory_replay(envs, golden, name):
    """Two epochs through the Trainer's FusedAdam on the recorded batches, each epoch on the masked adjacency of the
    recorded pruning draw: per-batch losses and per-epoch metrics."""
    gold = golden(f"traj_mmgcf_{name}_tiny.npz")
    fusion, weighting = M.TRAJ[name]
    config, train, valid, test, model = build("MMGCF", envs[False], M.overrides(fusion, weighting, 2, float(gold["dropout"])))
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
        model.masked_adj = model.pruner.adj_from_keep(torch.from_numpy(gold["keep_idx"][ep]).to(dev))
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


@pytest.mark.parametrize("name", ["mean_normalized", "concat_alpha", "text_mean_alpha"])
def test_mmgcf_topk_equals_mask_topk_of_predict(envs, name):
    from mmrec_b200 import ops
    fusion, weighting, layers, text_only = M.CASES[name]
    config, train, valid, test, model = build("MMGCF", envs[text_only], M.overrides(fusion, weighting, layers))
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


def _reference_loss(model, adj, interaction):
    """The reference's `calculate_loss` (mmgcf.py:258-284) as its own expressions on the device: torch.sparse.mm layers,
    full-table F.linear, the torch fusion, then the gathers."""
    import torch.nn.functional as F
    users, pos, neg = interaction[0], interaction[1], interaction[2]
    r, c, v = adj.coo()
    A = torch.sparse_coo_tensor(torch.stack([r.long(), c.long()]), v, (adj.n_rows, adj.n_cols))
    ego = torch.cat([model.user_embedding.weight, model.item_id_embedding.weight], dim=0)
    layers = [ego]
    for _ in range(model.n_ui_layers):
        ego = torch.sparse.mm(A, ego)
        layers.append(ego)
    ua, ia = torch.split(torch.stack(layers, dim=1).mean(dim=1), [model.n_users, model.n_items], dim=0)
    feats = []
    if model.v_feat is not None:
        feats.append(F.linear(model.image_embedding.weight, model.image_trs.weight, model.image_trs.bias))
    if model.t_feat is not None:
        feats.append(F.linear(model.text_embedding.weight, model.text_trs.weight, model.text_trs.bias))
    if model.fusion_mode == "concat":
        ia = model._concat_fusion(ia, feats)
    else:
        alpha = torch.sigmoid(model.mm_alpha) if model.weighting == "alpha" else None
        ia = M.torch_late_fuse(ia, feats[0] if model.v_feat is not None else None, feats[-1] if model.t_feat is not None else None,
                               model.fusion_mode, model.weighting, alpha=alpha)
    mf = model.bpr_loss(ua[users], ia[pos], ia[neg])
    reg = (model.user_embedding.weight[users].norm(2).pow(2) + model.item_id_embedding.weight[pos].norm(2).pow(2)
           + model.item_id_embedding.weight[neg].norm(2).pow(2)) / (2 * len(users))
    return mf + model.reg_weight * reg


@pytest.mark.parametrize("name", list(M.CASES))
def test_gathered_training_route_equals_the_full_table_expression(envs, golden, name):
    fusion, weighting, layers, text_only = M.CASES[name]
    config, train, valid, test, model = build("MMGCF", envs[text_only], M.overrides(fusion, weighting, layers))
    dev = config["device"]
    model.pre_epoch_processing()
    model.train()
    batch = torch.from_numpy(golden("mmgcf_tiny.npz")["batch"]).to(dev)
    res = []
    for fn in (model.calculate_loss, lambda b: _reference_loss(model, model.masked_adj, b)):
        model.zero_grad()
        loss = fn(batch)
        loss.backward()
        res.append((loss.item(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}))
    (l0, g0), (l1, g1) = res
    assert abs(l0 - l1) <= 2e-6 * abs(l1)
    assert set(g0) == set(g1)
    scale = max(g.norm().item() for g in g1.values())
    for k in g1:                                                         # biases: cancellation noise, see M.grad_errors
        assert (g0[k] - g1[k]).norm().item() <= 1e-4 * max(g1[k].norm().item(), 1e-3 * scale), k
