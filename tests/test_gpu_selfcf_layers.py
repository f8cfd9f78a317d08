"""SELFCFED_LGN with two dropped layers against the reference (the `l2_*` phase of tests/golden/selfcfed_lgn_tiny.npz):
the forward through both masked layers and the backward's chain on the mirrored bits, with the reference's draws replayed;
and the keep bits of an empty matrix."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import golden_io as G  # noqa: E402
import selfcf_golden  # noqa: E402
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


def test_selfcf_two_layers_match_reference(env, golden):
    gold = golden("selfcfed_lgn_tiny.npz")
    config, train, valid, test, model = build("SELFCFED_LGN", env, {"n_layers": 2})
    dev = config["device"]
    assert model.online_encoder.n_layers == 2
    assert G.same_init(model, gold) == [], "initial state differs from the reference"
    model.train()
    model.zero_grad()
    fwd = []
    orig = model.forward

    def spy(inputs):
        o = orig(inputs)
        fwd.append(o)
        return o
    model.forward = spy
    with selfcf_golden.Replay(gold["l2_loss_seed"]) as rep:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]).to(dev))
    del model.forward
    assert rep.digests == list(gold["l2_loss_draw_sha256"])
    assert rel(fwd[0][0], gold["l2_fwd_u_online"]) < 1e-6 and rel(fwd[0][2], gold["l2_fwd_i_online"]) < 1e-6
    loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy().reshape(-1), gold["l2_loss"], rtol=2e-6)
    named = dict(model.named_parameters())
    ref_grads = {k[8:]: gold[k] for k in gold.files if k.startswith("l2_grad.")}
    assert set(ref_grads) == {k for k, p in named.items() if p.grad is not None}
    for k, gref in ref_grads.items():
        assert rel(named[k].grad, gref) < 1e-5, f"grad {k}"


def test_keep_bits_of_an_empty_matrix_are_zero(env):
    from mmrec_b200 import ops
    e = torch.empty(0, device="cuda")
    i = torch.empty(0, dtype=torch.int32, device="cuda")
    keep, keep_t = ops.edge_keep_bits(e, 0.5, i, i)
    assert keep.numel() == 1 and keep_t.numel() == 1 and not keep.any() and not keep_t.any()
