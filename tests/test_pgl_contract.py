"""PGL without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins and the loss kernel by the
reference's torch expression on the gathered rows, against the golden files recorded from the reference's class
(tests/golden/make_golden_pgl.py).

Bit for bit: the initial weights, the parameter order, the RNG state after construction, the epoch's keep indices (the
reference's own CPU `torch.multinomial` draw) and the four dropout masks of a training step.  The loss, gradients, forward
outputs and scores agree to fp32 reorder error, and the metrics to within the evaluator's float64 rounding."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from contract import assert_metrics, run  # noqa: E402


def test_class_against_the_reference():
    r = run("pgl_contract_worker.py")
    assert r["init_identical"] and r["same_keep"]
    assert r["fwd_rel"] < 1e-5
    assert set(r["cases"]) == {"rw0.", "rw1."}
    for p, c in r["cases"].items():
        assert c["same_masks"], p
        assert c["loss_shape"] == [] and abs(c["loss"] - c["want_loss"]) <= 1e-6 * abs(c["want_loss"]), (p, c["loss"], c["want_loss"])
        assert c["grad_keys"] and max(c["grad_rel"].values()) < 1e-5, (p, c["grad_rel"])
    assert r["score_rel"] < 1e-5
    assert_metrics(r)


def test_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches at dropout 0 and reg_weight 0.1: each epoch's keep
    indices (drawn after the recorded seed), every batch loss and the per-epoch metrics."""
    r = run("pgl_contract_worker.py", "traj")
    assert r["same_keep"]
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
