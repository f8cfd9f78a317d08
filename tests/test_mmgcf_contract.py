"""MMGCF without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins (tests/mmgcf_contract_worker.py),
against the golden files recorded from the reference's class (tests/golden/make_golden_mmgcf.py).

Bit for bit: the initial weights, the pruning draw and the masked adjacency's values.  The forward, loss, gradients and
scores agree to fp32 reorder error (the stand-in propagation sums a row in the coalesced matrix's order), the metrics
exactly; two epochs of `Trainer._train_epoch` with pruning replay every draw, loss and metric."""
import pytest

from contract import assert_metrics, run


def test_mmgcf_class_against_the_reference_in_every_recorded_case():
    res = run("mmgcf_contract_worker.py", "model")
    assert len(res) == 11
    for name, r in res.items():
        assert r["init_identical"] and r["keep_equal"] and r["masked_vals_equal"], name
        assert r["fwd_rel"] < 1e-6, name
        assert abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"]), name
        assert r["grad_keys"] and r["grad_rel"] < 2e-4, name
        assert r["score_rel"] < 1e-5, name
        assert_metrics(r)


@pytest.mark.parametrize("name", ["mean_normalized", "concat_alpha"])
def test_mmgcf_two_epoch_trajectory_with_pruning(name):
    r = run("mmgcf_contract_worker.py", "traj:" + name)
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["keep_equal"] == [True, True]
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
