"""LATTICE without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins (tests/lattice_contract_worker.py),
against the golden files recorded from the reference's class (tests/golden/make_golden_lattice.py).

Bit for bit: the initial weights.  The losses, gradients (learned graph included) and scores agree to fp32 reorder error
(the stand-ins sum the sparse graphs in entry order, the reference its dense rows), the metrics exactly; two epochs of
`Trainer._train_epoch` replay every loss and metric."""
from contract import assert_metrics, run


def test_lattice_class_against_the_reference_in_every_recorded_case():
    res = run("lattice_contract_worker.py", "model")
    assert len(res) == 6
    for name, r in res.items():
        assert r["init_identical"], name
        assert r["loss_rel"] < 1e-5, name
        assert r["grad_keys"] and r["grad_rel"] < 1e-4, name
        assert r["score_rel"] < 1e-5, name
        assert_metrics(r)


def test_lattice_two_epoch_trajectory():
    r = run("lattice_contract_worker.py", "traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
