"""MMGCF's construction on the CPU: the modes it refuses, and for every recorded case the construction order (each
initial state bit for bit, `state_dict` keys and parameter order) against the digests recorded from the reference
(tests/golden/mmgcf_tiny.npz).  The graph builders run kernels, so they are stubbed here: they draw nothing at random."""
import os
import sys
import tempfile

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import mmgcf_golden as M  # noqa: E402
import golden_io as G  # noqa: E402


class _Pruner:
    def __init__(self, *a):
        self.edge_indices = self.edge_values = None


@pytest.fixture
def cpu_graphs(monkeypatch):
    from mmrec_b200 import graph
    monkeypatch.setattr(graph, "build_norm_adj", lambda *a, **k: None)
    monkeypatch.setattr(graph, "EdgePruner", _Pruner)


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    for text_only in (False, True):
        tmp = tempfile.mkdtemp(prefix="mmrec_mmgcf_host_")
        u, i, e, d, f = synth.SHAPES["tiny"]
        v, t = synth.make_features(i, f, seed=1)
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", synth.make_graph(u, i, e, seed=0), None if text_only else v, t)
        out[text_only] = os.path.join(tmp, "data") + "/"
    return out


def _build(data, over):
    from mmrec_b200.models.mmgcf import MMGCF
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import init_seed
    config = Config("MMGCF", "tiny", dict({"data_path": data, "gpu_id": 0, "use_gpu": False}, **over))
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    for k, v in over.items():
        if k in ("embedding_size", "feat_embed_dim"):
            config[k] = v
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return MMGCF(config, train)


@pytest.mark.parametrize("name", list(M.CASES))
def test_construction_order_and_state_dict_match_the_reference(cpu_graphs, data_dirs, golden, name):
    gold = golden("mmgcf_tiny.npz")
    fusion, weighting, layers, text_only = M.CASES[name]
    model = _build(data_dirs[text_only], M.overrides(fusion, weighting, layers))
    want = {str(k)[len(name) + len(".init_sha256."):]: str(gold[k]) for k in gold.files if str(k).startswith(name + ".init_sha256.")}
    assert G.init_digests(model) == want                    # same keys in the same order, same bits
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold[name + ".param_order"]]
    assert not model.image_embedding.weight.requires_grad if not text_only else not hasattr(model, "image_embedding")
    assert not model.text_embedding.weight.requires_grad
    assert hasattr(model, "mm_alpha") == (weighting == "alpha")
    if fusion == "concat":                                               # every concat layer exists, used or not
        assert hasattr(model, "all_concat_layer") and hasattr(model, "id_mm_concat_layer")
        assert hasattr(model, "mm_concat_layer") == (not text_only)
    if weighting == "alpha":
        assert next(iter(model.state_dict())) == "mm_alpha"


@pytest.mark.parametrize("over,what", [
    ({"fusion_mode": ["prod"]}, "fusion_mode"),
    ({"weighting": ["gated"]}, "weighting"),
    ({"fusion_mode": ["mean"], "feat_embed_dim": 32}, "feat_embed_dim"),
    ({"fusion_mode": ["sum"], "embedding_size": 48, "feat_embed_dim": 48}, "embedding_size"),
])
def test_refused_modes(cpu_graphs, data_dirs, over, what):
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError, match=what):
        _build(data_dirs[False], over)


def test_concat_takes_any_width(cpu_graphs, data_dirs):
    model = _build(data_dirs[False], {"fusion_mode": ["concat"], "weighting": ["equal"], "feat_embed_dim": 32})
    assert model.mm_concat_layer.weight.shape == (32, 64) and model.id_mm_concat_layer.weight.shape == (64, 96)
