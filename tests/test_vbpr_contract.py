"""VBPR and BPR without a GPU: the classes under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins and the loss kernel by the
reference's torch expression on the gathered rows, against the golden files recorded from the reference's classes
(tests/golden/make_golden_vbpr.py).

Bit for bit: the initial weights, the parameter order and the RNG state after construction.  The gathered projection
sums the weight gradient over 2B rows where the reference sums it over every item, and scatters in another order: the
loss, gradients and scores agree to fp32 reorder error, and the metrics to within the evaluator's float64 rounding."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import vbpr_golden as V  # noqa: E402
from contract import assert_metrics, run  # noqa: E402


@pytest.mark.parametrize("p", list(V.CASES))
def test_class_against_the_reference(p):
    r = run("vbpr_contract_worker.py", p)
    assert r["init_identical"]
    assert r["loss_shape"] == [1] and abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and max(r["grad_rel"].values()) < 1e-5, r["grad_rel"]
    assert r["score_rel"] < 1e-5
    assert_metrics(r)


@pytest.mark.parametrize("name", list(V.TRAJ))
def test_two_epoch_trajectory(name):
    """`Trainer._train_epoch` for two epochs on the recorded batches: every batch loss, the per-epoch metrics, and no
    torch RNG draw in any `calculate_loss`, here as in the reference."""
    r = run("vbpr_contract_worker.py", "traj:" + name)
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["rng_kept"]
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
