"""VBPR and BPR on the CPU: the configs, the construction order and RNG consumption (every initial state bit for bit
against the digests recorded from the reference, tests/golden/vbpr_tiny.npz and bpr_tiny.npz), the raw feature table, and
the refusals of the loss kernel's entry points, in the C ABI and in `ops.bpr_mf_loss`, before any CUDA call."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_io as G  # noqa: E402
import vbpr_golden as V  # noqa: E402


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    for mods in ("vt", "v", "t", ""):
        tmp = tempfile.mkdtemp(prefix="mmrec_vbpr_host_")
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", synth.named("tiny"), v if "v" in mods else None,
                            t if "t" in mods else None)
        out[mods] = os.path.join(tmp, "data") + "/"
    return out


def _config(name, data):
    from mmrec_b200.utils.configurator import Config
    return Config(name, "tiny", {"data_path": data, "gpu_id": 0, "use_gpu": False, "train_batch_size": 512})


def _build(name, data):
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    config = _config(name, data)
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return get_model(name)(config, train), config


@pytest.mark.parametrize("name", ["VBPR", "BPR"])
def test_config_takes_the_reference_keys_and_values(data_dirs, name):
    config = _config(name, data_dirs["vt"])
    assert config["embedding_size"] == 64 and config["hyper_parameters"][-1:] == ["reg_weight"]
    assert config["reg_weight"] == [2.0, 1.0, 1e-01, 1e-02, 1e-03, 1e-04, 1e-05]
    assert config["is_multimodal_model"] == (name == "VBPR")


@pytest.mark.parametrize("p", list(V.CASES))
def test_construction_order_and_rng_consumption_match_the_reference(data_dirs, golden, p):
    name, mods = V.CASES[p]
    gold = golden(f"{name.lower()}_tiny.npz")
    model, config = _build(name, data_dirs[mods])
    assert G.equal(gold, p + "rng_after_init", torch.get_rng_state().numpy())
    want = {str(k)[len(p + "init_sha256."):]: str(gold[k]) for k in gold.files if str(k).startswith(p + "init_sha256.")}
    assert G.init_digests(model) == want                    # same keys in the same order, same bits
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold[p + "param_order"]]
    assert list(gold[p + "cfg"]) == [str(config["embedding_size"]), str(config["reg_weight"])]
    if name == "VBPR":
        feats = [f for f in (model.t_feat, model.v_feat) if f is not None]      # text first
        assert torch.equal(model.item_raw_features, torch.cat(feats, -1))
        assert "item_raw_features" not in model.state_dict()
        assert model.u_embedding.shape == (model.n_users, 128)
        assert model.item_linear.weight.shape == (64, model.item_raw_features.shape[1])
        assert not hasattr(model, "get_item_embedding")


def test_c_entry_points_refuse_bad_arguments():
    from mmrec_b200 import _lib
    lib = _lib.load()
    P = 0x1000                                                           # a fake device address: nothing is dereferenced
    ws = lib.mmrec_bpr_mf_workspace_bytes(8)
    assert ws >= 16 and lib.mmrec_bpr_mf_workspace_bytes(0) == 0
    fwd = lib.mmrec_bpr_mf_f32
    assert fwd(0, 64, 64, 0, P, P, None, P, P, P, 1.0, P, P, P, P, ws, None) == -1         # B = 0
    assert b"bpr_mf" in lib.mmrec_last_error()
    assert fwd(8, 64, 32, 0, P, P, None, P, P, P, 1.0, P, P, P, P, ws, None) == -1         # du != da + dp
    assert fwd(8, 128, 64, 64, P, P, None, P, P, P, 1.0, P, P, P, P, ws, None) == -1       # dp > 0 without P
    assert fwd(8, 64, 64, 0, P, None, None, P, P, P, 1.0, P, P, P, P, ws, None) == -1      # da > 0 without A
    assert fwd(8, 64, 64, 0, P, P, None, None, P, P, 1.0, P, P, P, P, ws, None) == -1      # null users
    assert fwd(8, 64, 64, 0, P, P, None, P, P, P, 1.0, None, P, P, P, ws, None) == -1      # null loss
    assert fwd(8, 64, 64, 0, P, P, None, P, P, P, 1.0, P, P, P, P, ws - 1, None) == -2     # workspace too small
    assert b"workspace" in lib.mmrec_last_error()
    bwd = lib.mmrec_bpr_mf_bwd_f32
    assert bwd(8, 64, 64, 0, P, P, None, P, P, P, 1.0, P, P, None, P, P, None, None) == -1     # null g
    assert bwd(8, 64, 64, 0, P, P, None, P, P, P, 1.0, P, P, P, P, None, None, None) == -1     # da > 0 without gA_rows
    assert bwd(8, 128, 64, 64, P, P, P, P, P, P, 1.0, P, P, P, P, P, None, None) == -1        # dp > 0 without gP_rows
    assert bwd(-1, 64, 64, 0, P, P, None, P, P, P, 1.0, P, P, P, P, P, None, None) == -1      # negative B


def test_ops_bpr_mf_loss_refuses_bad_arguments():
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    U, A, Pr = torch.zeros(10, 128), torch.zeros(7, 64), torch.zeros(8, 64)
    i4 = torch.arange(4)
    for args in ((U, A, None, i4, i4, i4),                              # 128 != 64 + 0
                 (U, A, torch.zeros(8, 32), i4, i4, i4),               # 128 != 64 + 32
                 (U, A, torch.zeros(6, 64), i4, i4, i4),               # P is not [2B, dp]
                 (U, A, Pr, i4, i4, torch.arange(3)),                  # B differs
                 (U, A, Pr, i4[:0], i4[:0], i4[:0]),                   # B = 0
                 (U, A, Pr, i4.float(), i4, i4),                       # float indices
                 (U[0], A, Pr, i4, i4, i4)):                           # 1-D U
        with pytest.raises(MMRecError):
            ops.bpr_mf_loss(*args, 1.0)
    if not torch.cuda.is_available():
        with pytest.raises(MMRecError):
            ops.bpr_mf_loss(U, A, Pr, i4, i4, i4, 1.0)                  # CPU tensors: no CPU path
