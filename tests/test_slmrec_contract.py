"""SLMRec without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded
from the reference's class (tests/golden/make_golden_slmrec.py).

The stand-ins run the reference's own ops: `torch.sparse.mm` + stack + mean sums every column of the [N, 3d] ego table in
the order the three d-wide propagations do, so the views, tables, loss, scores and metrics match bit for bit.  One
gradient does not: `embedding_user.weight` feeds all three views, and autograd adds its three column-block gradients in
another order than the reference's three `torch.cat`s (fp32 reorder error, and through it the trajectory's later losses)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(arg):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "slmrec_contract_worker.py"), arg], capture_output=True, text=True,
                         timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.startswith("CONTRACT ")]
    assert out.returncode == 0 and lines, out.stdout[-3000:] + out.stderr[-3000:]
    return json.loads(lines[-1][len("CONTRACT "):])


def test_slmrec_class_against_the_reference():
    r = _run("model")
    assert r["init_identical"]
    assert all(r["views_equal"].values()) and r["tables_equal"]
    assert r["loss"] == r["want_loss"]
    assert r["grad_keys"]
    assert set(r["grad_rel"]) - set(r["grad_equal"]) <= {"embedding_user.weight"}
    assert max(r["grad_rel"].values()) < 1e-6
    assert r["score_equal"]
    for k, v in r["want_valid"].items():
        assert abs(r["valid"][k] - v) < 1e-9, (k, r["valid"][k], v)
    for k, v in r["want_test"].items():
        assert abs(r["test"][k] - v) < 1e-9, (k, r["test"][k], v)


def test_slmrec_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches: every batch loss and the per-epoch metrics."""
    r = _run("traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-6 and r["metric_max_abs"] < 1e-9
