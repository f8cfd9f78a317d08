"""SLMRec's three views as one width-3d SpMM (K1 at d in {96, 192, 384}) and the model class.

K1 at width 3d runs three float4 per lane on the lanes the width d uses, so every d-wide column block of the product is the
width-d product of that block, bit for bit, on any fp32 input: with and without the plan, on rows run by a whole CTA and on
split rows, for the Y output and the running-sum / mean epilogue, and on a transposed CSR.  (The cosine gate reduces over the
whole row, so its blocks are not separable: it is checked against torch.)  On exactly representable operands the product
equals float64, and repeated runs give the same bits.  Then the model against the golden files recorded from the reference
(tests/golden/make_golden_slmrec.py), and `full_sort_topk` against `mask_topk` of `full_sort_predict` where sigmoid
saturates."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

# empty rows, short rows, CTA-sized tasks, one segment, two segments (513, 520) and nine (4200)
ROW_LENS = [0, 0, 1, 7, 32, 33, 64, 511, 512, 513, 520, 4200, 0, 3]
N_COLS = 4500


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _matrix(dev, seed, exact=False, n_fill=300):
    from mmrec_b200.ops import CSR
    rng = np.random.default_rng(seed)
    lens = ROW_LENS + list(rng.integers(0, 40, n_fill))
    row = np.concatenate([np.full(n, r, dtype=np.int64) for r, n in enumerate(lens)])
    col = np.concatenate([np.sort(rng.choice(N_COLS, size=n, replace=False)) for n in lens]).astype(np.int64)
    if exact:
        vals = rng.integers(-3, 4, row.size).astype(np.float32) * np.float32(0.125)
    else:
        vals = rng.standard_normal(row.size).astype(np.float32)
    A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev), torch.from_numpy(vals).to(dev),
                     len(lens), N_COLS, sum_duplicates=False)
    assert A.n_split > 0 and A.n_cta_tasks > 0
    return A


def _run(A, X, epi, plan, acc_in):
    """"y": Y only; "acc": Y and the running sum / 3; "mean": the running sum only, / 4."""
    from mmrec_b200 import ops
    n, w = A.n_rows, X.shape[1]
    Y = torch.full((n, w), 7.0, device=X.device) if epi in ("y", "acc") else None
    acc_out = torch.full((n, w), 7.0, device=X.device) if epi in ("acc", "mean") else None
    div = {"y": 1.0, "acc": 3.0, "mean": 4.0}[epi]
    ops.spmm_raw(A, X, Y=Y, acc_in=acc_in if acc_out is not None else None, acc_out=acc_out, acc_div=div, use_plan=plan)
    return Y, acc_out


@pytest.mark.parametrize("plan", [True, False])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_column_blocks_equal_the_width_d_product(dev, d, plan):
    A = _matrix(dev, seed=d)
    for M in (A, A.t()):
        g = torch.Generator(device=dev).manual_seed(d)
        X = torch.randn(M.n_cols, 3 * d, device=dev, generator=g)
        acc_in = torch.randn(M.n_rows, 3 * d, device=dev, generator=g)
        for epi in ("y", "acc", "mean"):
            wide = _run(M, X, epi, plan, acc_in)
            for k in range(3):
                cols = slice(k * d, (k + 1) * d)
                narrow = _run(M, X[:, cols].contiguous(), epi, plan, acc_in[:, cols].contiguous())
                for a, b in zip(wide, narrow):
                    if a is not None:
                        assert torch.equal(a[:, cols], b), (d, plan, epi, k, M is A)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_width_3d_propagation_equals_three_propagations(dev, d):
    """`ops.propagate_mean` forward and backward on the [N, 3d] table against the three d-wide propagations, bit for bit,
    on a directed matrix (the backward runs on `CSR.t()`)."""
    from mmrec_b200 import ops
    A = _matrix(dev, seed=d + 7)
    from mmrec_b200.ops import CSR
    r, c, v = A.coo()
    keep = c < A.n_rows
    S = CSR.from_coo(r[keep], c[keep], v[keep], A.n_rows, A.n_rows, sum_duplicates=False)
    g = torch.Generator(device=dev).manual_seed(1)
    ego = torch.randn(S.n_rows, 3 * d, device=dev, generator=g).requires_grad_(True)
    w = torch.randn(S.n_rows, 3 * d, device=dev, generator=g)
    out = ops.propagate_mean(S, ego, 3)
    (out * w).sum().backward()
    for k in range(3):
        cols = slice(k * d, (k + 1) * d)
        e = ego.detach()[:, cols].contiguous().requires_grad_(True)
        o = ops.propagate_mean(S, e, 3)
        (o * w[:, cols].contiguous()).sum().backward()
        assert torch.equal(out.detach()[:, cols], o.detach()) and torch.equal(ego.grad[:, cols], e.grad)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_exact_operands_equal_float64_and_repeat(dev, d):
    A = _matrix(dev, seed=d + 1, exact=True)
    g = torch.Generator().manual_seed(d)
    X = (torch.randint(-7, 8, (N_COLS, 3 * d), generator=g).float() * 0.5).to(dev)
    acc_in = (torch.randint(-5, 6, (A.n_rows, 3 * d), generator=g).float() * 0.25).to(dev)
    r, c, v = A.coo()
    D = torch.zeros(A.n_rows, N_COLS, dtype=torch.float64, device=dev).index_put_((r, c), v.double(), accumulate=True)
    y64 = D @ X.double()
    for plan in (True, False):
        Y, acc = _run(A, X, "acc", plan, acc_in)
        assert torch.equal(Y.double(), y64)
        s = (acc_in.double() + y64).float().cpu()                           # exact in fp32; then one IEEE fp32 division
        assert torch.equal(acc.cpu(), s / torch.full_like(s, 3.0))
        Y2, acc2 = _run(A, X, "acc", plan, acc_in)
        assert torch.equal(Y, Y2) and torch.equal(acc, acc2)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_gate_at_width_3d(dev, d):
    """The cosine gate at width 3d reduces over the whole 3d row: against torch's expression."""
    from mmrec_b200 import ops
    A = _matrix(dev, seed=d + 2)
    g = torch.Generator(device=dev).manual_seed(3)
    X = torch.randn(N_COLS, 3 * d, device=dev, generator=g)
    ref = torch.randn(A.n_rows, 3 * d, device=dev, generator=g)
    Y = torch.empty(A.n_rows, 3 * d, device=dev)
    ops.spmm_raw(A, X, Y=Y, gate_ref=ref)
    r, c, v = A.coo()
    y = torch.zeros(A.n_rows, 3 * d, dtype=torch.float64, device=dev).index_add_(0, r, v.double().unsqueeze(1) * X.double()[c])
    want = torch.nn.functional.cosine_similarity(y, ref.double(), dim=-1, eps=1e-8).unsqueeze(1) * y
    assert (Y.double() - want).abs().max().item() < 1e-5 * want.abs().max().item()


# ----------------------------------------------------------------------------------------------------------------------
# the model class against the reference's golden files
# ----------------------------------------------------------------------------------------------------------------------
import golden_io as G  # noqa: E402
from test_gpu_models import build, rel  # noqa: E402


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


def test_slmrec_matches_reference(env, golden):
    from mmrec_b200._lib import MMRecError
    gold = golden("slmrec_tiny.npz")
    config, train, valid, test, model = build("SLMRec", env, {})
    dev = config["device"]
    assert G.same_init(model, gold) == [], "initial state differs from the reference"
    assert [k for k, _ in model.named_parameters()] == list(gold["param_order"])
    assert model.norm_adj.symmetric
    r, c, v = model.norm_adj.coo()
    idx = gold["adj_indices"]
    o = np.lexsort((idx[1], idx[0]))
    assert np.array_equal(torch.stack((r, c)).cpu().numpy(), idx[:, o])
    assert np.array_equal(v.cpu().numpy(), gold["adj_values"][o])
    model.eval()
    with pytest.raises(MMRecError):                                   # no training batch yet: no stored tables
        model.full_sort_predict([torch.zeros(1, dtype=torch.int64, device=dev)])
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    for name in ("i_emb", "v_emb", "t_emb"):
        assert rel(getattr(model, name).detach(), gold["view_" + name]) < 1e-6, name
    base = model.i_emb._base                                          # the views FAC reads are column blocks, not copies
    assert base is not None and all(getattr(model, n)._base is base for n in
                                    ("v_emb", "t_emb", "i_emb_u", "i_emb_i", "v_emb_u", "v_emb_i", "t_emb_u", "t_emb_i"))
    assert rel(model.all_users.detach(), gold["all_users"]) < 1e-5 and rel(model.all_items.detach(), gold["all_items"]) < 1e-5
    loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy().reshape(-1), gold["loss"], rtol=2e-6)
    named = dict(model.named_parameters())
    ref_grads = {k[5:]: gold[k] for k in gold.files if k.startswith("grad.")}
    assert set(ref_grads) == {k for k, p in named.items() if p.grad is not None}
    # the key-side biases of FAC's two logits (g_v_iv, g_t_ivat) have a gradient that is 0 in exact arithmetic (the rows of
    # a softmax cross-entropy gradient sum to 0): both sides hold rounding noise only
    noise = {"g_v_iv.bias", "g_t_ivat.bias"}
    for k, gref in ref_grads.items():
        if k in noise:
            assert np.abs(gref).max() < 1e-8 and named[k].grad.abs().max().item() < 1e-8, f"grad {k}"
        else:
            assert rel(named[k].grad, gref) < 1e-5, f"grad {k}"
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]).to(dev), torch.from_numpy(gold["eval_mask"]).to(dev)]
    with torch.no_grad():
        scores = model.full_sort_predict(eb)
        assert (scores.cpu() - torch.from_numpy(gold["scores"])).abs().max().item() < 1e-5
    from mmrec_b200.common.trainer import Trainer
    tr = Trainer(config, model)
    res = tr.evaluate(valid)
    np.testing.assert_allclose(np.array([res[k] for k in gold["metric_names"]]), gold["metric_values"], atol=1e-4 + 1e-12)
    res_t = tr.evaluate(test, is_test=True)
    np.testing.assert_allclose(np.array([res_t[k] for k in gold["metric_names"]]), gold["test_metric_values"], atol=1e-4 + 1e-12)


def test_slmrec_topk_ranks_the_sigmoid(env):
    """`full_sort_topk` = `mask_topk` of `full_sort_predict`, bit for bit, also where sigmoid saturates: there the tied
    items come in ascending index, as a stable sort of the sigmoid scores gives."""
    from mmrec_b200 import ops
    config, train, valid, test, model = build("SLMRec", env, {})
    dev = config["device"]
    model.train()
    model.calculate_loss(next(iter(train)).to(dev)).backward()
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid))
        eb = [eb[0].to(dev), eb[1].to(dev)]
        model.all_users = model.all_users.detach().clone()
        model.all_users[eb[0][:20]] *= 2000.0                         # scores of tens: sigmoid rounds many to 1.0
        idx = model.full_sort_topk(eb, 50)
        s = model.full_sort_predict(eb)
        assert int(((s == 1.0).sum(1) > 50).sum()) > 0, "no saturated row"
        _, want = ops.mask_topk(s.clone(), eb[1], 50)
        assert torch.equal(idx, want)
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10
        key = m.cpu().numpy()
        order = np.argsort(-key, axis=1, kind="stable")[:, :50]
        assert np.array_equal(idx.cpu().numpy(), order)


def test_slmrec_trajectory_replay(env, golden):
    """Two epochs through the Trainer's FusedAdam on the recorded batches: per-batch losses and per-epoch metrics."""
    gold = golden("traj_slmrec_tiny.npz")
    config, train, valid, test, model = build("SLMRec", env, {})
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
            loss = model.calculate_loss(batches[:, offs[b]:offs[b + 1]].to(dev))
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
