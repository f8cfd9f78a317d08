"""SELFCFED_LGN's host logic without a GPU: the reference's stored entry order of the normalised adjacency (the order its
dropout draws are applied in), the keep rule and scale against torch's CPU expression bit for bit, the golden files' draws,
an oracle restatement of the dropped propagation on the CPU against the reference's recorded forward, and the refusal of
CPU tensors."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import golden_io as G  # noqa: E402
from mmrec_b200 import graph  # noqa: E402


def _scipy_norm_adj(r, c, nu, ni):
    """`get_norm_adj_mat` of src/common/encoders.py:39-75, its COO (row, col, fp32 value) in stored order."""
    if not hasattr(sp.dok_matrix, "_update"):                         # private API gone from newer scipy: the dict update it did
        sp.dok_matrix._update = lambda self, d: self._dict.update({k: np.float32(v) for k, v in d.items()})
    inter = sp.coo_matrix((np.ones(r.size, np.float32), (r, c)), shape=(nu, ni))
    it = inter.transpose()
    A = sp.dok_matrix((nu + ni, nu + ni), dtype=np.float32)
    d = dict(zip(zip(inter.row, inter.col + nu), [1] * inter.nnz))
    d.update(dict(zip(zip(it.row + nu, it.col), [1] * it.nnz)))
    A._update(d)
    diag = np.power(np.array((A > 0).sum(axis=1).flatten())[0] + 1e-7, -0.5)
    D = sp.diags(diag)
    L = sp.coo_matrix(D * A * D)
    return L.row, L.col, L.data.astype(np.float32)


def _in_reference_order(r, c, nu, ni):
    rows, cols, vals = graph.norm_adj_entries(r, c, nu, ni)
    draw_of, mirror = graph.dropout_entry_maps(r, c, nu, ni)
    perm = np.empty_like(draw_of)
    perm[draw_of] = np.arange(draw_of.size, dtype=draw_of.dtype)
    return rows[perm], cols[perm], vals[perm], (rows, cols, mirror)


@pytest.mark.parametrize("seed", range(4))
def test_entry_order_equals_scipy(seed):
    """Random graphs with repeated (user, item) pairs in file order, and one in canonical order."""
    rng = np.random.default_rng(seed)
    nu, ni, m = 300, 200, 3000
    r, c = rng.integers(0, nu, m), rng.integers(0, ni, m)
    if seed == 3:
        o = np.lexsort((c, r))
        r, c = r[o], c[o]
    rr, cc, vv = _scipy_norm_adj(r, c, nu, ni)
    gr, gc, gv, (rows, cols, mirror) = _in_reference_order(r, c, nu, ni)
    assert np.array_equal(gr, rr) and np.array_equal(gc, cc) and np.array_equal(gv, vv)
    assert np.array_equal(rows[mirror], cols) and np.array_equal(cols[mirror], rows)


def _encoder_inter(gold):
    """The interaction COO as the encoder reads it: `inter_matrix(form='coo').astype(np.float32)` (encoders.py:15-16); with
    this scipy `astype` from the loader's float64 canonicalises it (sorted, repeated pairs summed)."""
    nu, ni = int(gold["n_users"]), int(gold["n_items"])
    m = sp.coo_matrix((np.ones(gold["inter_row"].size), (gold["inter_row"], gold["inter_col"])), shape=(nu, ni))
    m = m.astype(np.float32)
    return m.row, m.col, nu, ni


def test_entry_order_equals_the_golden_indices(golden):
    gold = golden("selfcfed_lgn_tiny.npz")
    r, c, v, _ = _in_reference_order(*_encoder_inter(gold))
    assert np.array_equal(np.stack([r, c]), gold["adj_indices"]) and np.array_equal(v, gold["adj_values"])


def _keep_np(kp, draws):
    """The mask kernel's rule: floorf(__fadd_rn(float32(1 - rate), r)) != 0."""
    return np.floor(np.float32(kp) + draws.astype(np.float32)) != 0


@pytest.mark.parametrize("rate", [0.0, 0.25, 0.5, 0.7071, 0.999999, 1e-9, 0.123456789])
def test_keep_rule_and_scale_equal_torch(rate):
    g = torch.Generator().manual_seed(1)
    draws = torch.rand(100000, generator=g)
    kp = np.float32(1 - rate)
    edge = np.float32(1) - kp
    near = np.array([np.nextafter(edge, np.float32(-1)), edge, np.nextafter(edge, np.float32(2))], dtype=np.float32)
    near = near[(near >= 0) & (near < 1)]
    draws[:near.size] = torch.from_numpy(near)
    random_tensor = 1 - np.float64(rate)                               # encoders.py:78-80, as the reference writes it
    random_tensor += draws
    want = torch.floor(random_tensor).type(torch.bool).numpy()
    assert np.array_equal(_keep_np(kp, draws.numpy()), want)
    vals = torch.rand(5000, generator=g)
    x = torch.sparse_coo_tensor(torch.stack((torch.arange(5000), torch.arange(5000))), vals, (5000, 5000))
    scaled = (x * (1. / (1 - np.float64(rate))))._values().numpy()
    assert np.array_equal(scaled, vals.numpy() * np.float32(1. / (1 - rate)))


def test_golden_draws_regenerate(golden):
    """The recorded phases regenerate from their seeds: the rate, `torch.rand(nnz)` and the two target masks."""
    import selfcf_golden
    gold = golden("selfcfed_lgn_tiny.npz")
    nnz = gold["adj_indices"].shape[1]
    rep = selfcf_golden.Replay(gold["loss_seed"])
    rep.seed_phase()
    assert np.random.random() == float(gold["loss_rate"])
    digests = [G.sha256_fp32(torch.rand(nnz).numpy())]
    B = gold["batch"].shape[1]
    for _ in range(2):
        digests.append(G.sha256_fp32(selfcf_golden.cpu_dropout_mask((B, int(gold["cfg_embedding_size"])), float(gold["cfg_dropout"])).numpy()))
    assert digests == list(gold["loss_draw_sha256"])


def test_dropped_propagation_oracle_matches_the_reference_forward(golden):
    """The CSR-order keep bits (draw_of, the keep rule, fp32 scale) restated with torch on the CPU reproduce the reference's
    recorded forward: the rows the recorded batch gathers from the dropped propagation of the initial weights."""
    import selfcf_golden
    gold = golden("selfcfed_lgn_tiny.npz")
    ir, ic, nu, ni = _encoder_inter(gold)
    rows, cols, vals = graph.norm_adj_entries(ir, ic, nu, ni)
    draw_of, _ = graph.dropout_entry_maps(ir, ic, nu, ni)
    # the initial weights the reference drew: init_seed(999) then xavier_uniform_ user, item (checked against the digests)
    from mmrec_b200.utils.utils import init_seed
    init_seed(999)
    torch.manual_seed(999)
    d = int(gold["cfg_embedding_size"])
    ue = torch.nn.init.xavier_uniform_(torch.empty(nu, d))
    ie = torch.nn.init.xavier_uniform_(torch.empty(ni, d))
    if G.sha256_fp32(ue.numpy()) != str(gold["init_sha256.param0.online_encoder.embedding_dict.user_emb"]):
        pytest.skip("the harness seeds differently from init_seed(999) + manual_seed here")
    assert G.sha256_fp32(ie.numpy()) == str(gold["init_sha256.param0.online_encoder.embedding_dict.item_emb"])
    rep = selfcf_golden.Replay(gold["loss_seed"])
    rep.seed_phase()
    rate = np.random.random()
    draws = torch.rand(rows.size).numpy()
    keep = _keep_np(np.float32(1 - rate), draws[draw_of])
    v = vals[keep] * np.float32(1. / (1 - rate))
    n = nu + ni
    A = torch.sparse_coo_tensor(torch.from_numpy(np.stack([rows[keep], cols[keep]])), torch.from_numpy(v), (n, n))
    x = torch.cat([ue, ie])
    layers = [x]
    for _ in range(int(gold["cfg_n_layers"])):
        x = torch.sparse.mm(A, x)
        layers.append(x)
    out = torch.stack(layers, 1).mean(1)
    b = torch.from_numpy(gold["batch"])
    assert torch.equal(out[:nu][b[0]], torch.from_numpy(gold["fwd_u_online"]))
    assert torch.equal(out[nu:][b[1]], torch.from_numpy(gold["fwd_i_online"]))


def test_cpu_tensors_are_refused():
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError):
        ops.edge_keep_bits(torch.rand(64), 0.5, torch.zeros(64, dtype=torch.int32))

    class Sym:
        symmetric = True
    with pytest.raises(MMRecError):
        ops.propagate_mean_dropped(Sym(), torch.zeros(4, 32), 2, torch.zeros(1, dtype=torch.int32),
                                   torch.zeros(1, dtype=torch.int32), 1.0)
