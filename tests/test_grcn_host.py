"""GRCN on the CPU: the config, the construction order and RNG consumption (every initial state bit for bit against the
digests recorded from the reference, tests/golden/grcn_tiny.npz), the refusals, the routing loop's reduction to repeated
normalisations on the reference's own expression (GATConv under the generator's PyG shim), and the attention graph's
edge-order map against the reference's `cat(edge_index, edge_index[[1, 0]])`.  The graph build runs kernels, so
construction stubs it here; it draws nothing at random."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_io as G  # noqa: E402
from make_golden_grcn import CASES, MessagePassing, softmax  # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "grcn_tiny.npz"), allow_pickle=True)


@pytest.fixture
def cpu_graphs(monkeypatch):
    from mmrec_b200 import graph
    monkeypatch.setattr(graph, "build_grcn_adj", lambda *a, **k: (None, None))


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    for mods in ("vt", "v", "t"):
        tmp = tempfile.mkdtemp(prefix="mmrec_grcn_host_")
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", synth.named("tiny"), v if "v" in mods else None,
                            t if "t" in mods else None)
        out[mods] = os.path.join(tmp, "data") + "/"
    return out


def _build(data, over):
    from mmrec_b200.models.grcn import GRCN
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import init_seed
    config = Config("GRCN", "tiny", dict({"data_path": data, "gpu_id": 0, "use_gpu": False, "train_batch_size": 512}, **over))
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return GRCN(config, train), train


def test_config_takes_the_reference_keys_and_values(data_dirs, gold):
    from mmrec_b200.utils.configurator import Config
    config = Config("GRCN", "tiny", {"data_path": data_dirs["vt"], "gpu_id": 0, "use_gpu": False})
    assert config["n_layers"] == 3 and config["hyper_parameters"][-2:] == ["reg_weight", "learning_rate"]
    assert config["reg_weight"] == [0.1, 0.01, 0.001, 0.0001, 0.00001]
    assert config["learning_rate"] == [1, 0.1, 0.01, 0.001, 0.0001]
    for k in ("embedding_size", "latent_embedding"):
        assert float(config[k]) == float(gold["cfg_" + k]), k
    assert config["reg_weight"][0] == float(gold["cfg_reg_weight"]) and config["learning_rate"][0] == float(gold["cfg_learning_rate"])


@pytest.mark.parametrize("p", list(CASES))
def test_construction_order_and_rng_consumption_match_the_reference(cpu_graphs, data_dirs, gold, p):
    over, mods = CASES[p]
    model, _ = _build(data_dirs[mods], dict(over))
    assert G.equal(gold, p + "rng_after_init", torch.get_rng_state().numpy())
    want = {str(k)[len(p + "init_sha256."):]: str(gold[k]) for k in gold.files
            if str(k).startswith(p + "init_sha256.") and (p or not any(str(k).startswith(q) for q in CASES if q))}
    assert G.init_digests(model) == want
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold[p + "param_order"]]
    assert "v_gcn.features" not in model.state_dict() and model.result.shape == (model.n_users + model.n_items, 64)


def test_refusals(cpu_graphs, data_dirs):
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError, match="conetent_rep"):
        _build(data_dirs["t"], {})
    with pytest.raises(MMRecError, match="no image features"):
        _build(data_dirs["vt"], {"is_multimodal_model": False})


class _GATConv(MessagePassing):
    """The reference's `GATConv.message` (src/models/grcn.py:61-73), restated for the shim's `propagate`."""

    def message(self, x_i, x_j, size_i, edge_index_i):
        self.alpha = softmax(torch.mul(x_i, x_j).sum(dim=-1), edge_index_i, num_nodes=size_i)
        return x_j * self.alpha.view(-1, 1)


@pytest.mark.parametrize("num_routing", [1, 3])
def test_routing_loop_is_repeated_normalisation(gold, num_routing):
    """`CGCN.forward`'s loop (`:149-156`) on the one-directional edge list: the aggregation reaches item rows only, so the
    user rows of `preference` are normalised num_routing more times and nothing else; values equal up to the sign of a
    zero, gradients equal bit for bit."""
    U, I = int(gold["n_users"]), int(gold["n_items"])
    edge_index = torch.stack([torch.from_numpy(gold["inter_row"]), torch.from_numpy(gold["inter_col"]) + U])
    g = torch.Generator().manual_seed(5)
    pref0 = torch.randn(U, 64, generator=g)
    pref0[0, :3] = -0.0
    feats = torch.randn(I, 64, generator=g)
    up = torch.randn(U, 64, generator=g)

    def reference(p):
        preference = F.normalize(p)
        features = F.normalize(feats)
        conv = _GATConv()
        for _ in range(num_routing):
            x = torch.cat((preference, features), dim=0)
            x_hat_1 = conv.propagate(edge_index, x=x)
            preference = preference + x_hat_1[:U]
            preference = F.normalize(preference)
        return preference

    def port(p):
        preference = F.normalize(p)
        for _ in range(num_routing):
            preference = F.normalize(preference)
        return preference

    outs, grads = [], []
    for fn in (reference, port):
        p = pref0.clone().requires_grad_(True)
        out = fn(p)
        (out * up).sum().backward()
        outs.append(out.detach())
        grads.append(p.grad)
    assert torch.equal(outs[0], outs[1])                              # == : +0 and -0 compare equal
    assert torch.equal(grads[0], grads[1])


def test_edge_order_map_is_the_reference_order(gold):
    """CSR position e of the attention graph holds the reference's edge order[e] of `cat(edge_index, edge_index[[1, 0]])`:
    rows are targets (`edge_index[1]`), columns sources, ascending, repeated edges in their reference order."""
    from mmrec_b200 import graph
    U, I = int(gold["n_users"]), int(gold["n_items"])
    r, c = np.append(gold["inter_row"], gold["inter_row"][0]), np.append(gold["inter_col"], gold["inter_col"][0])  # one repeat
    rows, cols, order = graph.grcn_edge_order(r, c, U, I)
    ei = np.stack([r, c + U])
    sym = np.concatenate([ei, ei[[1, 0]]], axis=1)
    assert np.array_equal(rows, sym[1][order]) and np.array_equal(cols, sym[0][order])
    assert np.array_equal(np.sort(order), np.arange(sym.shape[1]))
    key = rows * (U + I) + cols
    assert np.all(np.diff(key) >= 0)
    dup = np.flatnonzero(np.diff(key) == 0)
    assert dup.size == 2 and np.all(order[dup] < order[dup + 1])
    # the confidence gather: the source node's row, users for the forward edges, items for the reversed ones
    assert np.array_equal(cols, np.concatenate([ei[0], ei[1]])[order])
