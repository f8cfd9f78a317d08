"""DRAGON's construction on the CPU: the config, the refused modes, and for both modalities, text only and 'mean' the
construction order (each initial state bit for bit, `state_dict` keys, parameter order and the `np.random` / torch draws
that follow the constructor) against the digests recorded from the reference (tests/golden/dragon_tiny.npz,
make_golden_dragon.py).  The graph builders run kernels, so they are stubbed here: they draw nothing at random."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_io as G  # noqa: E402

CASES = {"": ({}, False), "text.": ({}, True), "mean.": ({"aggr_mode": ["mean"]}, False)}


class _Graph:
    def t(self):
        return self


@pytest.fixture
def cpu_graphs(monkeypatch):
    from mmrec_b200 import graph
    from mmrec_b200.models import dragon
    monkeypatch.setattr(graph, "build_freedom_mm_adj", lambda *a, **k: _Graph())
    monkeypatch.setattr(graph, "build_gcn_add_adj", lambda *a, **k: _Graph())
    monkeypatch.setattr(dragon, "mean_adj_from_edges", lambda *a, **k: _Graph())


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    for text_only in (False, True):
        tmp = tempfile.mkdtemp(prefix="mmrec_dragon_host_")
        u, i, e, d, f = synth.SHAPES["tiny"]
        g = synth.make_graph(u, i, e, seed=0)
        v, t = synth.make_features(i, f, seed=1)
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, None if text_only else v, t)
        synth.write_user_graph_dict(os.path.join(tmp, "data"), "tiny", g)
        out[text_only] = os.path.join(tmp, "data") + "/"
    return out


def _build(data, over):
    from mmrec_b200.models.dragon import DRAGON
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import init_seed
    config = Config("DRAGON", "tiny", dict({"data_path": data, "gpu_id": 0, "use_gpu": False, "train_batch_size": 512}, **over))
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return DRAGON(config, train)


def test_config_takes_the_reference_keys_and_values(data_dirs):
    from mmrec_b200.utils.configurator import Config
    config = Config("DRAGON", "tiny", {"data_path": data_dirs[False], "gpu_id": 0, "use_gpu": False})
    want = {"embedding_size": 64, "feat_embed_dim": 64, "n_mm_layers": 1, "n_layers": 2, "knn_k": 10, "mm_image_weight": 0.1,
            "aggr_mode": ["add"], "learning_rate": [0.1, 0.01, 0.001, 0.0001, 0.00001],
            "reg_weight": [0.1, 0.01, 0.001, 0.0001, 0.00001]}
    for k, v in want.items():
        assert config[k] == v, k
    assert config["hyper_parameters"][-3:] == ["aggr_mode", "reg_weight", "learning_rate"]   # after the overall seed


@pytest.mark.parametrize("p", list(CASES))
def test_construction_order_and_state_dict_match_the_reference(cpu_graphs, data_dirs, golden, p):
    gold = golden("dragon_tiny.npz")
    over, text_only = CASES[p]
    model = _build(data_dirs[text_only], over)
    np_after, torch_after = np.random.randint(0, 2 ** 31, 4).astype(np.int64), torch.randint(0, 2 ** 31, (4,)).numpy()
    want = {str(k)[len(p + "init_sha256."):]: str(gold[k]) for k in gold.files if str(k).startswith(p + "init_sha256.")}
    assert G.init_digests(model) == want                    # same keys in the same order, same bits
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold[p + "param_order"]]
    assert "result_embed" not in dict(model.named_parameters())
    assert model.result_embed.dtype == torch.float64 and model.result_embed.shape == (model.n_users + model.n_items, 64)
    assert model.MLP_user.weight.shape == (64, 128)
    assert model.v_preference is None and model.t_preference is None
    assert np.array_equal(np_after, gold[p + "rng_after_np"])            # the reference's RNG stream is consumed
    assert np.array_equal(torch_after, gold[p + "rng_after_torch"])
    assert model.construction == "cat" and model.aggr_mode == str(gold[p + "cfg_aggr_mode"])


@pytest.mark.parametrize("over,what", [
    ({"aggr_mode": ["max"]}, "aggr_mode"),
    ({"aggr_mode": [""]}, "aggr_mode"),
])
def test_refused_modes(cpu_graphs, data_dirs, over, what):
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError, match=what):
        _build(data_dirs[False], over)


def test_the_model_never_reads_or_writes_the_mm_adj_file(cpu_graphs, data_dirs):
    path = os.path.join(data_dirs[False], "tiny", "mm_adj_10.pt")
    torch.save("not a graph", path)                                      # a stale file the reference would load
    try:
        _build(data_dirs[False], {})
        assert torch.load(path) == "not a graph"
    finally:
        os.remove(path)
    _build(data_dirs[False], {})
    assert not os.path.exists(path)
