"""GRCN without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded
from the reference's class (tests/golden/make_golden_grcn.py).

Bit for bit: the initial weights, the parameter order and the RNG state after construction.  The stand-ins run PyG's
gathers and scatters on the attention graph's CSR order, where the reference scatters in its edge order: the
representation, loss, gradients and scores agree to fp32 reorder error, and the metrics exactly."""
from contract import assert_metrics, run


def _check_model(r):
    assert r["init_identical"]
    assert r["pre_score_rel"] < 1e-6 and r["representation_rel"] < 1e-6
    assert r["loss_shape"] == [1] and abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and max(r["grad_rel"].values()) < 1e-5
    assert r["score_rel"] < 1e-5
    assert_metrics(r)


def test_grcn_class_against_the_reference():
    _check_model(run("grcn_contract_worker.py", "model"))


def test_grcn_one_routing_layer_against_the_reference():
    _check_model(run("grcn_contract_worker.py", "l1"))


def test_grcn_image_only_against_the_reference():
    _check_model(run("grcn_contract_worker.py", "image"))


def test_grcn_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches: every batch loss and the per-epoch metrics."""
    r = run("grcn_contract_worker.py", "traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
