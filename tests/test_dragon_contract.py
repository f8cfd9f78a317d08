"""DRAGON without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded
from the reference's class (tests/golden/make_golden_dragon.py), with the dataset's user graph written by
`synth.write_user_graph_dict`.

Bit for bit: the initial weights and float64 `result_embed`, the float64 scores before any forward, the epoch's user-graph
sample and the mutated batch.  Large tensors are compared through fixed random sketches (tests/golden/golden_io.py).
The stand-ins sum a row's neighbours in the coalesced sparse matrix's order and the user graph's duplicates are coalesced,
where the reference scatters edge by edge and runs a batched matmul: `user_rep`, loss, gradients and scores agree to fp32
reorder error, and the metrics exactly."""
from contract import assert_metrics, run


def _check_model(r):
    assert r["init_identical"]
    assert r["scores0_equal"] and r["sample_equal"] and r["batch_after_equal"]
    assert r["user_rep_rel"] < 1e-6 and r["result_embed_rel"] < 1e-6
    assert abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and max(r["grad_rel"].values()) < 1e-5
    assert r["score_rel"] < 1e-5
    assert_metrics(r)


def test_dragon_class_against_the_reference():
    r = run("dragon_contract_worker.py", "model")
    assert r["has_v_gcn"]
    _check_model(r)


def test_dragon_text_only_against_the_reference():
    r = run("dragon_contract_worker.py", "text")
    assert not r["has_v_gcn"]
    _check_model(r)


def test_dragon_mean_aggregation_against_the_reference():
    r = run("dragon_contract_worker.py", "mean")
    assert r["has_v_gcn"]
    _check_model(r)


def test_dragon_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches, `np.random` seeded before each epoch's sample: every
    batch loss and the per-epoch metrics."""
    r = run("dragon_contract_worker.py", "traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
