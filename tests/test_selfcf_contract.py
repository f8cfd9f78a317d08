"""SELFCFED_LGN without a GPU: the class (and its encoder `LightGCN_Encoder`) under the harness the reference's quick_start
builds (its own code with MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the
golden files recorded from the reference's class (tests/golden/make_golden_selfcf.py).  The class draws the rate, the edge
dropout and the target masks itself from the seeded CPU generators; the draws are compared by digest."""
from contract import assert_metrics, run


def _check_loss_phase(r, n_layers):
    assert r["init_identical"] and r["n_layers"] == n_layers
    assert r["draws_ok"] and 0 < r["n_kept"] < r["nnz"]
    # the stand-in propagation is the reference's own expression on the same kept entries: the forward rows bit for bit
    assert r["fwd_u_equal"] and r["fwd_i_equal"]
    assert abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and r["grad_rel"] < 1e-6


def test_selfcf_class_against_the_reference():
    """Initial weights bit for bit (their SHA-256) in the reference's parameter order; the same draws; forward rows, loss and
    gradients; first-batch scores (one width-2d product against the reference's two products and an add: fp32 reorder
    error); the valid / test metrics of `Trainer.evaluate`."""
    r = run("selfcf_contract_worker.py", "model")
    _check_loss_phase(r, 1)
    assert r["score_err"] < 1e-5
    assert_metrics(r)


def test_selfcf_two_layers_against_the_reference():
    """The class built with `n_layers` = 2: two dropped layers forward and the backward through both."""
    _check_loss_phase(run("selfcf_contract_worker.py", "layers2"), 2)


def test_selfcf_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches, each seeded as recorded: every batch's draws and loss,
    and the per-epoch metrics."""
    r = run("selfcf_contract_worker.py", "traj")
    assert r["n_batches"] == r["want_batches"] == 8 and r["draws_ok"]
    assert r["loss_max_rel"] < 1e-6 and r["metric_max_abs"] < 1e-9
