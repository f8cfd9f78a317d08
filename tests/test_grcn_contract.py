"""GRCN without a GPU: the class under the harness the reference's quick_start builds (its own code with
MMREC_REFERENCE_SRC, else the package's restatement), kernels replaced by CPU stand-ins, against the golden files recorded
from the reference's class (tests/golden/make_golden_grcn.py).

Bit for bit: the initial weights, the parameter order and the RNG state after construction.  The stand-ins run PyG's
gathers and scatters on the attention graph's CSR order, where the reference scatters in its edge order: the
representation, loss, gradients and scores agree to fp32 reorder error, and the metrics exactly."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(arg):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "grcn_contract_worker.py"), arg], capture_output=True, text=True,
                         timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.startswith("CONTRACT ")]
    assert out.returncode == 0 and lines, out.stdout[-3000:] + out.stderr[-3000:]
    return json.loads(lines[-1][len("CONTRACT "):])


def _check_model(r):
    assert r["init_identical"]
    assert r["pre_score_rel"] < 1e-6 and r["representation_rel"] < 1e-6
    assert r["loss_shape"] == [1] and abs(r["loss"] - r["want_loss"]) <= 1e-6 * abs(r["want_loss"])
    assert r["grad_keys"] and max(r["grad_rel"].values()) < 1e-5
    assert r["score_rel"] < 1e-5
    for k, v in r["want_valid"].items():
        assert abs(r["valid"][k] - v) < 1e-9, (k, r["valid"][k], v)
    for k, v in r["want_test"].items():
        assert abs(r["test"][k] - v) < 1e-9, (k, r["test"][k], v)


def test_grcn_class_against_the_reference():
    _check_model(_run("model"))


def test_grcn_one_routing_layer_against_the_reference():
    _check_model(_run("l1"))


def test_grcn_image_only_against_the_reference():
    _check_model(_run("image"))


def test_grcn_two_epoch_trajectory():
    """`Trainer._train_epoch` for two epochs on the recorded batches: every batch loss and the per-epoch metrics."""
    r = _run("traj")
    assert r["n_batches"] == r["want_batches"] == 8
    assert r["loss_max_rel"] < 1e-5 and r["metric_max_abs"] < 1e-9
