"""SELFCFED_LGN's edge dropout inside K1 (`mmrec_spmm_op.keep_bits`, `mmrec_edge_keep_bits`) and the model class.

The masked SpMM is checked bit for bit against the unmasked kernel on the compacted matrix (the kept entries, values
fl(v * scale)) on exactly representable operands (integers times a power of two, every partial sum exact: see
test_gpu_exact_arith.py), so summation order cannot hide an error: every width, with and without the plan, split rows of
several segments, every epilogue and rows with every entry dropped.  Then the mirrored bits against the compacted matrix's
transpose, the keep bits against torch's expression on the device, general inputs against the reference's expression
(`sparse_dropout` + `torch.sparse.mm`), gradients against torch autograd, run-to-run bit equality, and the model against
the golden files recorded from the reference (tests/golden/make_golden_selfcf.py) with its draws replayed."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def unpack_bits(keep, nnz):
    e = torch.arange(nnz, device=keep.device)
    return ((keep[e >> 5] >> (e & 31).to(torch.int32)) & 1).bool()


def pack_bits(mask):
    nnz = mask.numel()
    m = torch.zeros(((nnz + 31) // 32) * 32, dtype=torch.int64, device=mask.device)
    m[:nnz] = mask.to(torch.int64)
    w = (m.view(-1, 32) << torch.arange(32, device=mask.device)).sum(1)
    return (w - (w >= 2 ** 31).to(torch.int64) * 2 ** 32).to(torch.int32)


def compacted(A, keep_mask, scale):
    from mmrec_b200.ops import CSR
    r, c, v = A.coo()
    k = keep_mask[:A.nnz]
    vals = v[k] * torch.tensor(scale, dtype=torch.float32, device=v.device)   # one fp32 multiply per kept value
    return CSR.from_coo(r[k], c[k], vals, A.n_rows, A.n_cols, sum_duplicates=False, symmetric=False)


# ----------------------------------------------------------------------------------------------------------------------
# exactly representable operands
# ----------------------------------------------------------------------------------------------------------------------
# empty rows, a lane-group row, a CTA-sized task, one segment, 513 / 520 (two segments) and 4200 (nine segments)
ROW_LENS = [0, 0, 1, 7, 32, 33, 64, 511, 512, 513, 520, 4200, 0, 3]
N_COLS = 4500
V_UNIT, X_UNIT = 2.0 ** -3, 2.0 ** -1


def _exact_matrix(dev, seed, n_fill=300):
    """CSR of integer values (|v| <= 3, units of 1/8) and the rows whose every entry the test drops."""
    from mmrec_b200.ops import CSR
    rng = np.random.default_rng(seed)
    lens = ROW_LENS + list(rng.integers(0, 40, n_fill))
    row = np.concatenate([np.full(n, r, dtype=np.int64) for r, n in enumerate(lens)])
    col = np.concatenate([np.sort(rng.choice(N_COLS, size=n, replace=False)) for n in lens]).astype(np.int64)
    vals = rng.integers(-3, 4, row.size).astype(np.float32)
    vals[vals == 0] = 1
    A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev), torch.from_numpy(vals * V_UNIT).to(dev),
                     len(lens), N_COLS, sum_duplicates=False)
    return A, torch.from_numpy(row).to(dev)


def _exact_x(dev, n, d, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-7, 8, (n, d), generator=g).float() * X_UNIT).to(dev)


def _run(A, X, epi, drop=None, plan=True):
    """One SpMM with epilogue `epi`: "y" (Y only), "acc" (Y and the running sum / 3), "mean" (running sum only, / 4)."""
    from mmrec_b200 import ops
    n, d = A.n_rows, X.shape[1]
    g = torch.Generator().manual_seed(5)
    acc_in = (torch.randint(-5, 6, (n, d), generator=g).float() * 0.25).to(X.device)
    Y = torch.full((n, d), 7.0, device=X.device) if epi in ("y", "acc") else None
    acc_out = torch.full((n, d), 7.0, device=X.device) if epi in ("acc", "mean") else None
    div = {"y": 1.0, "acc": 3.0, "mean": 4.0}[epi]
    ops.spmm_raw(A, X, Y=Y, acc_in=acc_in if acc_out is not None else None, acc_out=acc_out, acc_div=div, use_plan=plan, drop=drop)
    return Y, acc_out


@pytest.mark.parametrize("plan", [True, False])
@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_drop_equals_compacted_exact(dev, d, plan):
    A, row = _exact_matrix(dev, seed=d)
    assert A.n_split > 0 and A.n_cta_tasks > 0                         # split rows and CTA tasks are exercised
    X = _exact_x(dev, N_COLS, d, seed=d + 1)
    g = torch.Generator(device=dev).manual_seed(d)
    keep = torch.rand(A.nnz, generator=g, device=dev) < 0.6
    keep &= ~((row == 7) | (row == 11) | (row == 3))                  # rows of 511, 4200 and 7 entries lose all of them
    bits = pack_bits(keep)
    for scale in (2.0, 0.5, 1.0):
        C = compacted(A, keep, scale)
        for epi in ("y", "acc", "mean"):
            got = _run(A, X, epi, drop=(bits, scale), plan=plan)
            want = _run(C, X, epi, plan=plan)
            for a, b in zip(got, want):
                if a is not None:
                    assert torch.equal(a, b), (d, plan, scale, epi)
        Y, _ = _run(A, X, "y", drop=(bits, scale), plan=plan)
        assert not Y[7].any() and not Y[11].any() and not Y[3].any()


def test_drop_rate_zero_is_the_unmasked_kernel(dev):
    """rate = 0: every draw is kept (1 + r >= 1) and the scale is 1: the unmasked product bit for bit, general inputs."""
    from mmrec_b200 import graph, ops
    A, draw_of, mirror, nnz = _sym_graph(dev, 2000, 900, 30000, seed=3)
    ego = torch.randn(A.n_rows, 64, device=dev)
    keep, keep_t = ops.edge_keep_bits(torch.rand(nnz, device=dev), 1.0, draw_of, mirror)
    assert bool(unpack_bits(keep, nnz).all()) and bool(unpack_bits(keep_t, nnz).all())
    a = ops.propagate_mean_dropped(A, ego, 3, keep, keep_t, 1.0)
    b = ops.propagate_mean(A, ego, 3)
    assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------------------------
# the symmetric normalised adjacency: mirrored bits, keep rule, reference expression, gradients
# ----------------------------------------------------------------------------------------------------------------------
def _sym_graph(dev, n_users, n_items, n_edges, seed):
    from mmrec_b200 import graph
    rng = np.random.default_rng(seed)
    u = rng.integers(0, n_users, n_edges)
    i = (rng.pareto(1.2, n_edges) * 20).astype(np.int64) % n_items    # power-law items: split rows
    A = graph.build_norm_adj((u, i), n_users, n_items, dev)
    draw_of, mirror = graph.dropout_entry_maps(u, i, n_users, n_items)
    return A, torch.from_numpy(draw_of).to(dev), torch.from_numpy(mirror).to(dev), A.nnz


def _reference_matrix(A, draw_of, draws, rate):
    """`sparse_dropout` of encoders.py:77-88 on the device, on the entries in the reference's stored order."""
    r, c, v = A.coo()
    perm = torch.empty_like(draw_of)
    perm[draw_of.long()] = torch.arange(A.nnz, device=v.device, dtype=perm.dtype)
    idx = torch.stack((r[perm.long()], c[perm.long()]))
    x = torch.sparse_coo_tensor(idx, v[perm.long()], (A.n_rows, A.n_cols))
    random_tensor = 1 - rate
    random_tensor += draws
    mask = torch.floor(random_tensor).type(torch.bool)
    out = torch.sparse_coo_tensor(x._indices()[:, mask], x._values()[mask], x.shape)
    return out * (1. / (1 - rate)), mask


def test_keep_bits_equal_torch_on_the_device(dev):
    from mmrec_b200 import ops
    A, draw_of, mirror, nnz = _sym_graph(dev, 3000, 1000, 40000, seed=1)
    rng = np.random.default_rng(0)
    for rate in [0.0, 0.37, 0.5, 0.999, float(rng.random()), float(rng.random())]:
        kp = np.float32(1 - rate)
        draws = torch.rand(nnz, device=dev)
        edge = np.float32(1) - kp                                      # the draws around the rounding boundary
        near = np.array([np.nextafter(edge, np.float32(0)), edge, np.nextafter(edge, np.float32(1))], dtype=np.float32)
        near = near[(near >= 0) & (near < 1)]
        draws[:near.size * 50] = torch.from_numpy(np.tile(near, 50)).to(dev)
        _, ref_mask = _reference_matrix(A, draw_of, draws, rate)
        keep, keep_t = ops.edge_keep_bits(draws, float(kp), draw_of, mirror)
        got = unpack_bits(keep, nnz)
        assert torch.equal(got, ref_mask[draw_of.long()]), rate
        assert torch.equal(unpack_bits(keep_t, nnz), got[mirror.long()]), rate
        if nnz % 32:                                                   # bits past nnz are 0
            assert (keep[-1].item() & 0xFFFFFFFF) >> (nnz % 32) == 0


def test_mirrored_bits_are_the_transpose(dev):
    """The product with the mirrored bits equals the compacted dropped matrix's `CSR.t()`, bit for bit (exact values)."""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    A0, draw_of, mirror, nnz = _sym_graph(dev, 3000, 1000, 40000, seed=2)
    r, c, _ = A0.coo()
    sym_v = (((r + c) % 7) - 3).float()
    sym_v[sym_v == 0] = 1
    A = CSR(A0.n_rows, A0.n_cols, A0.rowptr, A0.colidx, (sym_v * V_UNIT).contiguous(), nnz, symmetric=True)
    X = _exact_x(dev, A.n_rows, 64, seed=9)
    keep, keep_t = ops.edge_keep_bits(torch.rand(nnz, device=dev), float(np.float32(1 - 0.5)), draw_of, mirror)
    C = compacted(A, unpack_bits(keep, nnz), 2.0)
    got = torch.empty_like(X)
    ops.spmm_raw(A, X, Y=got, drop=(keep_t, 2.0))
    want = torch.empty_like(X)
    ops.spmm_raw(C.t(), X, Y=want)
    assert torch.equal(got, want)


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_general_inputs_against_the_reference_expression(dev, d):
    """fp32 inputs: within reorder tolerance of the compacted route (split rows: other segment boundaries) and of the
    reference's `torch.sparse.mm` chain on the device; the gradient against torch autograd through that chain."""
    from mmrec_b200 import ops
    A, draw_of, mirror, nnz = _sym_graph(dev, 4000, 1500, 60000, seed=d)
    assert A.n_split > 0
    rate = 0.3141
    draws = torch.rand(nnz, device=dev)
    kp, scale = float(np.float32(1 - rate)), float(np.float32(1. / (1 - rate)))
    keep, keep_t = ops.edge_keep_bits(draws, kp, draw_of, mirror)
    ego = torch.randn(A.n_rows, d, device=dev, requires_grad=True)
    out = ops.propagate_mean_dropped(A, ego, 2, keep, keep_t, scale)
    C = compacted(A, unpack_bits(keep, nnz), scale)
    ref_c = ops.propagate_mean(C, ego.detach(), 2)
    tol = 1e-5 * out.abs().max().item()
    assert (out.detach() - ref_c).abs().max().item() < tol
    R, _ = _reference_matrix(A, draw_of, draws, rate)
    e = ego.detach().clone().requires_grad_(True)
    layers = [e]
    x = e
    for _ in range(2):
        x = torch.sparse.mm(R, x)
        layers.append(x)
    ref = torch.stack(layers, 1).mean(1)
    assert (out.detach() - ref.detach()).abs().max().item() < tol
    w = torch.randn_like(ref)
    (out * w).sum().backward()
    (ref * w).sum().backward()
    assert (ego.grad - e.grad).abs().max().item() < 1e-5 * e.grad.abs().max().item()


def test_bit_reproducible(dev):
    from mmrec_b200 import ops
    A, draw_of, mirror, nnz = _sym_graph(dev, 4000, 1500, 60000, seed=11)
    draws = torch.rand(nnz, device=dev)
    keep, keep_t = ops.edge_keep_bits(draws, 0.75, draw_of, mirror)
    outs = []
    for _ in range(3):
        ego = torch.randn(A.n_rows, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(0)).requires_grad_(True)
        y = ops.propagate_mean_dropped(A, ego, 3, keep, keep_t, float(np.float32(1 / 0.75)))
        y.square().sum().backward()
        outs.append((y.detach(), ego.grad))
    k2 = ops.edge_keep_bits(draws, 0.75, draw_of, mirror)
    assert torch.equal(keep, k2[0]) and torch.equal(keep_t, k2[1])
    for y, gx in outs[1:]:
        assert torch.equal(y, outs[0][0]) and torch.equal(gx, outs[0][1])


def test_unsupported_width_is_an_error(dev):
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    A, draw_of, mirror, nnz = _sym_graph(dev, 300, 100, 2000, seed=0)
    keep, keep_t = ops.edge_keep_bits(torch.rand(nnz, device=dev), 0.5, draw_of, mirror)
    with pytest.raises(MMRecError):
        ops.propagate_mean_dropped(A, torch.randn(A.n_rows, 48, device=dev), 2, keep, keep_t, 2.0)


# ----------------------------------------------------------------------------------------------------------------------
# the model class against the reference's golden files
# ----------------------------------------------------------------------------------------------------------------------
import golden_io as G  # noqa: E402
import selfcf_golden  # noqa: E402
from test_gpu_models import build, check_topk, rel  # noqa: E402


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


def test_selfcf_matches_reference(env, golden):
    gold = golden("selfcfed_lgn_tiny.npz")
    config, train, valid, test, model = build("SELFCFED_LGN", env, {})
    dev = config["device"]
    assert G.same_init(model, gold) == [], "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == list(gold["param_order"])
    enc = model.online_encoder
    r, c, v = enc.sparse_norm_adj.coo()
    perm = torch.empty_like(enc.draw_of)
    perm[enc.draw_of.long()] = torch.arange(enc.sparse_norm_adj.nnz, device=dev, dtype=perm.dtype)
    assert np.array_equal(torch.stack((r, c))[:, perm.long()].cpu().numpy(), gold["adj_indices"])
    assert np.array_equal(v[perm.long()].cpu().numpy(), gold["adj_values"])
    model.train()
    model.zero_grad()
    fwd = []
    orig = model.forward

    def spy(inputs):
        o = orig(inputs)
        fwd.append(o)
        return o
    model.forward = spy
    with selfcf_golden.Replay(gold["loss_seed"]) as rep:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    del model.forward
    assert rep.digests == list(gold["loss_draw_sha256"])
    assert rel(fwd[0][0], gold["fwd_u_online"]) < 1e-6 and rel(fwd[0][2], gold["fwd_i_online"]) < 1e-6
    loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy().reshape(-1), gold["loss"], rtol=2e-6)
    named = dict(model.named_parameters())
    ref_grads = {k[5:]: gold[k] for k in gold.files if k.startswith("grad.")}
    assert set(ref_grads) == {k for k, p in named.items() if p.grad is not None}
    for k, gref in ref_grads.items():
        assert rel(named[k].grad, gref) < 1e-5, f"grad {k}"
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


def test_selfcf_trajectory_replay(env, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches with the reference's draws: per-batch losses and
    per-epoch metrics."""
    gold = golden("traj_selfcfed_lgn_tiny.npz")
    config, train, valid, test, model = build("SELFCFED_LGN", env, {})
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.optim import FusedAdam
    trainer = Trainer(config, model)
    assert isinstance(trainer.optimizer, FusedAdam)
    dev = config["device"]
    batches = torch.from_numpy(gold["batches"])
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    names = list(gold["metric_names"])
    b = 0
    for ep, nb in enumerate(gold["batches_per_epoch"]):
        model.pre_epoch_processing()
        model.train()
        for _ in range(int(nb)):
            trainer.optimizer.zero_grad()
            with selfcf_golden.Replay(int(gold["seed0"]) + b) as rep:
                loss = model.calculate_loss(batches[:, offs[b]:offs[b + 1]].to(dev))
            assert rep.digests == list(gold["draw_sha256"][b])
            np.testing.assert_allclose(loss.item(), gold["losses"][b], rtol=5e-5)
            loss.backward()
            trainer.optimizer.step()
            b += 1
        trainer.lr_scheduler.step()
        v = trainer.evaluate(valid)
        t = trainer.evaluate(test, is_test=True)
        np.testing.assert_allclose([v[k] for k in names], gold["valid"][ep], atol=2e-4)
        np.testing.assert_allclose([t[k] for k in names], gold["test"][ep], atol=2e-4)
    assert b == int(gold["n_steps"])
