"""SLMRec without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded
from the reference's class (tests/golden/make_golden_slmrec.py).

The stand-ins run the reference's own ops: `torch.sparse.mm` + stack + mean sums every column of the [N, 3d] ego table in
the order the three d-wide propagations do, so the views, tables, loss, scores and metrics match bit for bit.  One
gradient does not: `embedding_user.weight` feeds all three views, and autograd adds its three column-block gradients in
another order than the reference's three `torch.cat`s (fp32 reorder error, and through it the trajectory's later losses)."""
from contract import assert_metrics, run


def test_slmrec_class_against_the_reference():
    r = run("slmrec_contract_worker.py", "model")
    assert r["init_identical"]
    assert all(r["views_equal"].values()) and r["tables_equal"]
    assert r["loss"] == r["want_loss"]
    assert r["grad_keys"]
    assert set(r["grad_rel"]) - set(r["grad_equal"]) <= {"embedding_user.weight"}
    assert max(r["grad_rel"].values()) < 1e-6
    assert r["score_equal"]
    assert_metrics(r)


def test_slmrec_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches: every batch loss and the per-epoch metrics."""
    r = run("slmrec_contract_worker.py", "traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-6 and r["metric_max_abs"] < 1e-9
