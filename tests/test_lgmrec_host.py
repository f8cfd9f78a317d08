"""LGMRec without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded from
the reference's class (tests/golden/make_golden_lgmrec.py) under the reference's own RNG stream; and the argument errors of
K8's entry points (include/mmrec_b200.h)."""
import os

import pytest
import torch

from contract import assert_metrics, run


@pytest.mark.parametrize("gfile", ["lgmrec_tiny.npz", "lgmrec_clothing_tiny.npz"])
def test_lgmrec_class_against_the_reference(gfile):
    """Initial weights bit for bit and in the reference's parameter order, `num_inters`, the same Gumbel / dropout draws in
    every phase, forward, loss, gradients, first-batch scores and the valid / test metrics of `Trainer.evaluate`."""
    r = run("lgmrec_contract_worker.py", gfile)
    assert r["init_identical"] and r["graphs"] and r["draws_ok"]
    assert r["fwd_rel"] < 1e-6 and r["grad_rel"] < 1e-5 and r["score_err"] < 1e-6
    assert abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert_metrics(r)


def test_lgmrec_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches and draws: every batch loss and the per-epoch metrics."""
    r = run("lgmrec_contract_worker.py", "traj")
    assert r["n_batches"] == 8 and r["draws_left"] == 0
    assert r["loss_max_rel"] < 1e-6 and r["metric_max_abs"] < 1e-9


def test_lgmrec_needs_both_modalities(tmp_path):
    from mmrec_b200.models.lgmrec import LGMRec

    class Cfg(dict):
        def __getitem__(self, k):
            return self.get(k)

    class DS:
        class dataset:
            get_user_num = staticmethod(lambda: 3)
            get_item_num = staticmethod(lambda: 2)
    import numpy as np
    os.makedirs(tmp_path / "x")
    np.save(tmp_path / "x" / "image_feat.npy", np.ones((2, 8), dtype=np.float32))
    cfg = Cfg(USER_ID_FIELD="u", ITEM_ID_FIELD="i", NEG_PREFIX="neg_", train_batch_size=2, device="cpu", end2end=False,
              is_multimodal_model=True, data_path=str(tmp_path) + "/", dataset="x", vision_feature_file="image_feat.npy",
              text_feature_file="text_feat.npy")
    with pytest.raises(ValueError, match="both modality"):
        LGMRec(cfg, DS())


def test_expsum_op_rejects_cpu_tensors():
    from mmrec_b200 import ops
    with pytest.raises(ops.MMRecError):
        ops.expsum_rows(torch.zeros(4, 64), torch.zeros(5, 64), 0.2)


def test_expsum_argument_errors_without_a_gpu():
    from mmrec_b200 import _lib
    lib = _lib.load()
    X = 16                                                            # never dereferenced: the checks come first
    assert lib.mmrec_expsum_rows_workspace_bytes(2048, 7050, 48) == 0          # d outside {32, 64, 128}
    assert lib.mmrec_expsum_rows_workspace_bytes(-1, 7050, 64) == 0
    assert lib.mmrec_expsum_rows_workspace_bytes(2048, 250000, 64) < 64 << 20  # O((B + M) d)
    assert lib.mmrec_expsum_rows_f32(4, X, 48, 5, X, 48, 48, 5.0, X, X, 1 << 20, None) == -1       # bad d
    assert b"expsum_rows" in lib.mmrec_last_error()
    assert lib.mmrec_expsum_rows_f32(-1, X, 64, 5, X, 64, 64, 5.0, X, X, 1 << 20, None) == -1      # negative B
    assert lib.mmrec_expsum_rows_f32(4, X, 64, -5, X, 64, 64, 5.0, X, X, 1 << 20, None) == -1      # negative M
    assert lib.mmrec_expsum_rows_f32(4, None, 64, 5, X, 64, 64, 5.0, X, X, 1 << 20, None) == -1    # null Q
    assert lib.mmrec_expsum_rows_f32(4, X, 64, 5, None, 64, 64, 5.0, X, X, 1 << 20, None) == -1    # null T
    assert lib.mmrec_expsum_rows_f32(4, X, 64, 5, X, 64, 64, 5.0, None, X, 1 << 20, None) == -1    # null ttl
    assert lib.mmrec_expsum_rows_f32(4, X, 32, 5, X, 64, 64, 5.0, X, X, 1 << 20, None) == -1       # ldq < d
    assert lib.mmrec_expsum_rows_f32(0, None, 64, 5, None, 64, 64, 5.0, None, None, 0, None) == -1  # M > 0 needs T
    assert lib.mmrec_expsum_rows_f32(0, None, 64, 0, None, 64, 64, 5.0, None, None, 0, None) == 0   # nothing to do
    assert lib.mmrec_expsum_rows_f32(4, X, 64, 5, X, 64, 64, 5.0, X, X, 0, None) == -2             # workspace too small
    bwd = lib.mmrec_expsum_rows_bwd_f32
    assert bwd(4, X, 64, 5, X, 64, 128 + 1, 5.0, X, X, 129, X, 129, X, 1 << 20, None) == -1         # bad d
    assert bwd(4, X, 64, 5, X, 64, 64, 5.0, X, None, 64, None, 64, X, 1 << 20, None) == -1          # no output requested
    assert bwd(4, X, 64, 5, X, 64, 64, 5.0, None, X, 64, X, 64, X, 1 << 20, None) == -1             # null g
    assert bwd(-4, X, 64, 5, X, 64, 64, 5.0, X, X, 64, X, 64, X, 1 << 20, None) == -1               # negative B
    assert bwd(4, X, 64, 5, X, 64, 64, 5.0, X, X, 63, X, 64, X, 1 << 20, None) == -1                # lddq < d
    assert bwd(4, X, 64, 5, X, 64, 64, 5.0, X, X, 64, X, 64, None, 0, None) == -1                   # null workspace
