"""MVGAE without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded from
the reference's class (tests/golden/make_golden_mvgae.py) under the reference's own RNG stream."""
import os

import pytest
import torch

from contract import assert_metrics, run


def test_mvgae_class_against_the_reference():
    """Initial weights and plain tensors bit for bit (their SHA-256), in the reference's parameter order; the same dropout masks and Gaussian
    noise; forward, the four decodes (values, and the argmax except at near ties), loss, gradients of every Parameter that
    gets one, first-batch scores of the cached `result_embed`, and the valid / test metrics of `Trainer.evaluate`."""
    r = run("mvgae_contract_worker.py", "model")
    assert r["init_identical"] and r["draws_ok"]
    assert r["fwd_rel"] < 1e-6
    assert r["n_decodes"] == 4 and r["decode_rel"] < 1e-6 and r["argmax_near_ties"]
    assert abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and r["grad_rel"] < 1e-5
    assert r["score_err"] < 1e-6
    assert_metrics(r)


def test_mvgae_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches and draws: every batch loss and the per-epoch metrics
    (scored from the last training forward's `result_embed`, as the reference does)."""
    r = run("mvgae_contract_worker.py", "traj")
    assert r["n_batches"] == 8 and r["draws_left"] == 0
    assert r["loss_max_rel"] < 1e-6 and r["metric_max_abs"] < 1e-9


def test_mvgae_needs_both_modalities(tmp_path):
    from mmrec_b200.models.mvgae import MVGAE

    class Cfg(dict):
        def __getitem__(self, k):
            return self.get(k)

    class DS:
        class dataset:
            get_user_num = staticmethod(lambda: 3)
            get_item_num = staticmethod(lambda: 2)
    import numpy as np
    os.makedirs(tmp_path / "x")
    np.save(tmp_path / "x" / "text_feat.npy", np.ones((2, 8), dtype=np.float32))
    cfg = Cfg(USER_ID_FIELD="u", ITEM_ID_FIELD="i", NEG_PREFIX="neg_", train_batch_size=2, device="cpu", end2end=False,
              is_multimodal_model=True, data_path=str(tmp_path) + "/", dataset="x", vision_feature_file="image_feat.npy",
              text_feature_file="text_feat.npy", embedding_size=4, n_layers=1, beta=0.1)
    with pytest.raises(ValueError, match="both modality"):
        MVGAE(cfg, DS())


def test_max_dot_rejects_cpu_tensors():
    from mmrec_b200 import ops
    with pytest.raises(ops.MMRecError):
        ops.max_dot(torch.zeros(4, 64), torch.zeros(5, 64))
