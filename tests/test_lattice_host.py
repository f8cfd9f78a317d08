"""LATTICE on the CPU: the config, the refusals, the construction order (every initial state bit for bit against the
digests recorded from the reference, tests/golden/lattice_tiny.npz), `norm_adj`'s builder bit for bit, and sparse
restatements of the original and learned graphs -- the kNN entries, the union, the weighted sums and the entry-wise
normalisation the model runs on the device -- against the reference's dense graphs, within the fp32 reordering bound (the
dense CPU sums add in another order).  The graph builders run kernels, so construction stubs them here; they draw
nothing at random.  No `image_adj_{k}.pt` / `text_adj_{k}.pt` is read or written."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_io as G  # noqa: E402
from make_golden_lattice import CASES  # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "lattice_tiny.npz"), allow_pickle=True)


@pytest.fixture
def cpu_graphs(monkeypatch):
    from mmrec_b200 import graph
    monkeypatch.setattr(graph, "build_lattice_norm_adj", lambda *a, **k: None)
    monkeypatch.setattr(graph, "build_mgcn_knn_adj", lambda *a, **k: None)

    def refuse(*a, **k):
        raise AssertionError("LATTICE must not read or write a .pt file")
    monkeypatch.setattr(torch, "load", refuse)
    monkeypatch.setattr(torch, "save", refuse)


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    for mods in ("vt", "v", "t"):
        tmp = tempfile.mkdtemp(prefix="mmrec_lattice_host_")
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", synth.make_graph(u, i, e, seed=0), v if "v" in mods else None,
                            t if "t" in mods else None)
        out[mods] = os.path.join(tmp, "data") + "/"
    return out


def _build(data, over):
    from mmrec_b200.models.lattice import LATTICE
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import init_seed
    config = Config("LATTICE", "tiny", dict({"data_path": data, "gpu_id": 0, "use_gpu": False, "train_batch_size": 512}, **over))
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return LATTICE(config, train), train


def test_config_takes_the_reference_keys_and_values(data_dirs, gold):
    from mmrec_b200.utils.configurator import Config
    config = Config("LATTICE", "tiny", {"data_path": data_dirs["vt"], "gpu_id": 0, "use_gpu": False})
    assert config["weight_size"] == [64, 64] and config["mess_dropout"] == [0.1, 0.1]
    assert config["cf_model"] == "lightgcn" and config["n_layers"] == 1 and config["knn_k"] == 10
    assert config["learning_rate_scheduler"] == [0.96, 50] and config["hyper_parameters"][-2:] == ["reg_weight", "learning_rate"]
    for k in ("embedding_size", "feat_embed_dim", "knn_k", "lambda_coeff"):
        assert float(config[k]) == float(gold["cfg_" + k]), k
    assert config["reg_weight"][0] == float(gold["cfg_reg_weight"]) and config["learning_rate"][0] == float(gold["cfg_learning_rate"])


@pytest.mark.parametrize("p", list(CASES))
def test_construction_order_and_initial_state_match_the_reference(cpu_graphs, data_dirs, gold, p):
    over, mods = CASES[p]
    model, _ = _build(data_dirs[mods], dict(over))
    want = {str(k)[len(p + "init_sha256."):]: str(gold[k]) for k in gold.files
            if str(k).startswith(p + "init_sha256.") and (p or not any(str(k).startswith(q) for q in CASES if q))}
    assert G.init_digests(model) == want
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold[p + "param_order"]]


def test_refusals(cpu_graphs, data_dirs):
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError, match="cf_model"):
        _build(data_dirs["vt"], {"cf_model": "gcn"})
    with pytest.raises(MMRecError, match="knn_k"):
        _build(data_dirs["vt"], {"knn_k": 121})


def test_no_adjacency_file_is_read_or_written(cpu_graphs, data_dirs):
    """A stale `image_adj_10.pt` / `text_adj_10.pt` beside the data is neither loaded nor replaced (`torch.load` /
    `torch.save` raise for the whole construction)."""
    root = os.path.join(data_dirs["vt"], "tiny")
    for name in ("image_adj_10.pt", "text_adj_10.pt"):
        with open(os.path.join(root, name), "wb") as f:
            f.write(b"not a graph")
    before = sorted(os.listdir(root))
    _build(data_dirs["vt"], {})
    assert sorted(os.listdir(root)) == before
    for name in ("image_adj_10.pt", "text_adj_10.pt"):
        with open(os.path.join(root, name), "rb") as f:
            assert f.read() == b"not a graph"
        os.remove(os.path.join(root, name))


def test_norm_adj_builder_is_the_reference_bit_for_bit(gold):
    from mmrec_b200 import graph
    rows, cols, vals = graph.lattice_norm_adj_entries(gold["inter_row"], gold["inter_col"], int(gold["n_users"]), int(gold["n_items"]))
    assert np.array_equal(np.stack([rows, cols]), gold["norm_adj_indices"])
    assert vals.dtype == np.float32 and np.array_equal(vals, gold["norm_adj_values"])


def test_norm_adj_builder_keeps_repeated_interactions():
    """The reference's lil assignment keeps a repeated (user, item) pair's multiplicity as the entry's value."""
    from mmrec_b200 import graph
    rows, cols, vals = graph.lattice_norm_adj_entries([0, 0, 1], [0, 0, 1], 2, 2)
    dense = np.zeros((4, 4))
    dense[rows, cols] = vals
    A = np.eye(4)
    A[0, 2] = A[2, 0] = 2.0
    A[1, 3] = A[3, 1] = 1.0
    want = (A / A.sum(1, keepdims=True)).astype(np.float32)
    assert np.array_equal(dense.astype(np.float32), want)


def _dense(gold, key, n):
    out = torch.zeros(n, n, dtype=torch.float64)
    out[tuple(torch.from_numpy(gold[key + ".index"]).long())] = torch.from_numpy(gold[key + ".values"]).double()
    return out


def _knn_entries(feat, k):
    """(row, col, value) of the cosine kNN, ties to the lower index: the entries of `build_knn_neighbourhood`."""
    cn = feat.div(torch.norm(feat, p=2, dim=-1, keepdim=True))
    val, ind = torch.topk(cn @ cn.t(), k, dim=-1)
    n = feat.shape[0]
    return torch.arange(n).repeat_interleave(k), ind.reshape(-1), val.reshape(-1)


def _sym_norm(r, c, a, n):
    rowsum = torch.zeros(n, dtype=a.dtype).index_add_(0, r, a)
    d = rowsum.pow(-0.5)
    d[torch.isinf(d)] = 0.0
    return (d[r] * a) * d[c]


def _to_dense(r, c, v, n):
    return torch.zeros(n, n, dtype=torch.float64).index_put_((r, c), v.double(), accumulate=True)


def _close(got, want, tol):
    assert torch.equal(got != 0, want != 0)
    assert (got - want).abs().max().item() <= tol * want.abs().max().item()


def test_original_graphs_sparse_restatement_against_the_reference(gold):
    from mmrec_b200.utils import synth
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    for feat, key in ((v, "image_original_adj"), (t, "text_original_adj")):
        r, c, a = _knn_entries(torch.from_numpy(np.asarray(feat, dtype=np.float32)), 10)
        _close(_to_dense(r, c, _sym_norm(r, c, a, i), i), _dense(gold, key, i), 1e-6)


@pytest.mark.parametrize("p", ["", "image.", "text."])
def test_learned_graph_sparse_restatement_against_the_reference(cpu_graphs, data_dirs, gold, p):
    """The graph-building batch's `item_adj` from the initial weights: kNN entries of each modality, their union with the
    original graphs' entries, fl(fl(w0 a) + fl(w1 b)), the entry-wise normalisation and the lambda mix."""
    over, mods = CASES[p]
    model, _ = _build(data_dirs[mods], dict(over))
    n, k, lam = model.n_items, model.knn_k, model.lambda_coeff
    w = torch.softmax(model.modal_weight.detach(), 0)
    learned = []
    with torch.no_grad():
        for m, trs, emb in (("v", "image_trs", "image_embedding"), ("t", "text_trs", "text_embedding")):
            if m in mods:
                feats = getattr(model, trs)(getattr(model, emb).weight)
                learned.append(_knn_entries(feats, k))
    originals = [(_dense(gold, key, n)) for m, key in (("v", "image_original_adj"), ("t", "text_original_adj")) if m in mods]
    keys = torch.cat([r * n + c for r, c, _ in learned] + [o.nonzero()[:, 0] * n + o.nonzero()[:, 1] for o in originals])
    uniq, inv = torch.unique(keys, return_inverse=True)
    parts = torch.split(inv, [x[0].numel() for x in learned] + [int((o != 0).sum()) for o in originals])
    vals = []
    for j, (_, _, a) in enumerate(learned):
        x = torch.zeros(uniq.numel())
        x[parts[j]] = a if len(learned) == 1 else w[j] * a
        vals.append(x)
    lv = vals[0] if len(vals) == 1 else vals[0] + vals[1]
    r, c = uniq // n, uniq % n
    L = _sym_norm(r, c, lv, n)
    ov = []
    for j, o in enumerate(originals):
        x = torch.zeros(uniq.numel())
        x[parts[len(learned) + j]] = o[o != 0].float()
        ov.append(x if len(originals) == 1 else w[j] * x)
    o_all = ov[0] if len(ov) == 1 else ov[0] + ov[1]
    item = (1 - lam) * L + lam * o_all
    _close(_to_dense(r, c, item, n), _dense(gold, p + "item_adj" if p + "item_adj.index" in gold.files else "item_adj", n), 1e-5)
