"""PGL on the CPU: the config, the construction order and RNG consumption (every initial state bit for bit against the
digests recorded from the reference, tests/golden/pgl_tiny.npz), the construction-time refusals, and the refusals of the
loss kernel's entry points, in the C ABI and in `ops.pgl_loss`, before any CUDA call."""
import os
import sys
import tempfile

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import golden_io as G  # noqa: E402


@pytest.fixture(scope="module")
def data_dirs():
    from mmrec_b200.utils import synth
    out = {}
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    for mods in ("vt", "v", "t"):
        tmp = tempfile.mkdtemp(prefix="mmrec_pgl_host_")
        synth.write_dataset(os.path.join(tmp, "data"), "tiny", synth.named("tiny"), v if "v" in mods else None,
                            t if "t" in mods else None)
        out[mods] = os.path.join(tmp, "data") + "/"
    return out


@pytest.fixture
def cpu_ops():
    """The graph builds of the construction on the CPU: tests/contract.py's stand-ins, put back afterwards."""
    sys.path.insert(0, HERE)
    import contract
    from mmrec_b200 import graph, ops
    saved = [(mod, dict(vars(mod))) for mod in (ops, graph)]
    contract.install_cpu_ops()
    yield
    for mod, d in saved:
        for k in [k for k in vars(mod) if k not in d]:
            delattr(mod, k)
        for k, v in d.items():
            setattr(mod, k, v)


def _config(data, **over):
    from mmrec_b200.utils.configurator import Config
    return Config("PGL", "tiny", dict({"data_path": data, "gpu_id": 0, "use_gpu": False, "train_batch_size": 512}, **over))


def _build(data, **after):
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    config = _config(data)
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    for k, v in after.items():
        config[k] = v
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    return get_model("PGL")(config, train), config


def test_config_takes_the_reference_keys_and_values(data_dirs):
    c = _config(data_dirs["vt"])
    assert c["hyper_parameters"][-3:] == ["dropout", "reg_weight", "mode"]
    assert (c["embedding_size"], c["feat_embed_dim"], c["weight_size"]) == (64, 64, [64, 64])
    assert (c["learning_rate_scheduler"], c["lambda_coeff"], c["learning_rate"]) == ([0.96, 50], 0.9, 0.001)
    assert (c["reg_weight"], c["dropout"], c["mode"]) == ([0], [0.2], ["local"])
    assert (c["n_mm_layers"], c["n_ui_layers"], c["knn_k"], c["mm_image_weight"]) == (1, 2, 10, 0.1)


def test_construction_order_and_rng_consumption_match_the_reference(data_dirs, golden, cpu_ops):
    gold = golden("pgl_tiny.npz")
    model, config = _build(data_dirs["vt"])
    assert G.equal(gold, "rng_after_init", torch.get_rng_state().numpy())
    want = {str(k)[len("init_sha256."):]: str(gold[k]) for k in gold.files if str(k).startswith("init_sha256.")}
    assert G.init_digests(model) == want                    # same keys in the same order, same bits
    assert [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    assert [k for k, _ in model.named_parameters()][:2] == ["user_text.weight", "user_image.weight"]
    assert model.dropoutf.p == 0.2 and model.reg_weight == 0 and model.mode == "local"
    assert not hasattr(model, "alignment") and not hasattr(model, "uniformity")


def test_epoch_keeps_the_reference_length(data_dirs, golden, cpu_ops):
    """`pre_epoch_processing` draws int(nnz * 0.3) edges: the recorded keep indices after the recorded seed."""
    gold = golden("pgl_tiny.npz")
    model, _ = _build(data_dirs["vt"])
    kept, orig = [], model.pruner.sample
    model.pruner.sample = lambda *a, **k: kept.append(orig(*a, **k)[1]) or (None, kept[-1])
    import pgl_golden as P
    torch.manual_seed(P.PRUNE_SEED)
    model.pre_epoch_processing()
    assert kept[0].numel() == int(model.edge_values.numel() * 0.3)
    assert torch.equal(kept[0], torch.from_numpy(gold["keep_idx"]))


@pytest.mark.parametrize("mods,after,what", [("vt", {"mode": "global"}, "sparsesvd"), ("v", {}, "both"), ("t", {}, "both"),
                                             ("vt", {"feat_embed_dim": 32}, "feat_embed_dim")])
def test_refusals(data_dirs, cpu_ops, mods, after, what):
    from mmrec_b200._lib import MMRecError
    with pytest.raises(MMRecError, match=what):
        _build(data_dirs[mods], **after)


def test_c_entry_points_refuse_bad_arguments():
    from mmrec_b200 import _lib
    lib = _lib.load()
    P = 0x1000                                                           # a fake device address: nothing is dereferenced
    rows = lib.mmrec_pgl_rows_f32
    m4 = (P, P, P, P)
    assert rows(0, 128, P, P, P, P, P, *m4, 1.25, P, P, P, P, P, P, P, None) == -1           # B = 0
    assert b"pgl_rows" in lib.mmrec_last_error()
    assert rows(8, 0, P, P, P, P, P, *m4, 1.25, P, P, P, P, P, P, P, None) == -1             # d = 0
    assert rows(8, 128, None, P, P, P, P, *m4, 1.25, P, P, P, P, P, P, P, None) == -1        # null UA
    assert rows(8, 128, P, P, P, P, P, P, None, P, P, 1.25, P, P, P, P, P, P, P, None) == -1  # three masks
    assert rows(8, 128, P, P, P, P, P, *m4, 1.25, None, P, P, P, P, P, P, None) == -1        # null x
    assert rows(8, 128, P, P, P, P, P, *m4, 1.25, P, P, None, P, P, P, P, None) == -1        # views incomplete
    fin = lib.mmrec_pgl_finish_f32
    assert fin(0, P, None, None, None, 0.0, P, None) == -1                                   # B = 0
    assert fin(8, P, P, P, None, 0.1, P, None) == -1                                         # ttl2 missing
    assert fin(8, P, None, None, None, 0.0, None, None) == -1                                # null loss
    fb = lib.mmrec_pgl_finish_bwd_f32
    assert fb(8, P, None, None, None, 0.0, None, P, None, None, None) == -1                   # null g
    assert fb(8, P, P, P, P, 0.1, P, P, P, None, None) == -1                                 # gttl missing
    rb = lib.mmrec_pgl_rows_bwd_f32
    assert rb(8, 128, P, P, P, P, P, *m4, 1.25, 1.25, None, None, None, None, None, None, None, P, P, None) == -1   # null gx
    assert rb(8, 128, P, P, P, P, P, *m4, 1.25, 1.25, P, P, P, P, P, P, None, P, P, None) == -1         # gvd missing
    assert rb(8, 128, P, P, P, P, P, *m4, 1.25, 1.25, P, None, None, None, None, None, None, P, None, None) == -1  # null gI


def test_ops_pgl_loss_refuses_bad_arguments():
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    UA, IA = torch.zeros(10, 128), torch.zeros(7, 128)
    i4 = torch.arange(4)
    mk = [torch.ones(4, 128, dtype=torch.bool)] * 4
    for args in ((UA, torch.zeros(7, 64), i4, i4, i4, mk),                  # widths differ
                 (UA, IA, i4, i4, torch.arange(3), mk),                     # B differs
                 (UA, IA, i4[:0], i4[:0], i4[:0], None),                    # B = 0
                 (UA, IA, i4.float(), i4, i4, mk),                          # float indices
                 (UA[0], IA, i4, i4, i4, mk),                               # 1-D UA
                 (UA, IA, i4, i4, i4, mk[:3]),                              # three masks
                 (UA, IA, i4, i4, i4, [torch.ones(4, 64, dtype=torch.bool)] * 4),   # mask shape
                 (UA, IA, i4, i4, i4, [torch.ones(4, 128)] * 4)):           # float masks
        with pytest.raises(MMRecError):
            ops.pgl_loss(*args, 0.2, 0.1)
    if not torch.cuda.is_available():
        with pytest.raises(MMRecError):
            ops.pgl_loss(UA, IA, i4, i4, i4, mk, 0.2, 0.1)                  # CPU tensors: no CPU path


def test_dropout_scales():
    """The forward scale is fp32(1 / fp32(1 - p)) (ATen's fused dropout), the backward's fp32(1 / (1 - p))."""
    import numpy as np
    from mmrec_b200 import ops
    assert ops.dropout_scales(0.2) == (1.25, 1.25)
    f, b = ops.dropout_scales(0.1)
    assert f == float(np.float32(1 / float(np.float32(0.9)))) and b == float(np.float32(1 / 0.9))
    assert ops.dropout_scales(1.0) == (0.0, 0.0)
