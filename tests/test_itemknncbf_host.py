"""ItemKNNCBF without a GPU: the CPU restatement (tests/itemknncbf_oracle.py) against the golden file recorded from the
reference's class (tests/golden/make_golden_itemknncbf.py); the class under the quick_start-built harness with CPU stand-ins
for K7's shrink route and K9; K9's ranking rule against a dense ranking on crafted rows; the argument errors of the new
entry points."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import itemknncbf_oracle as KO  # noqa: E402
from contract import assert_metrics, run  # noqa: E402

PREFIXES = ["s10_", "s0_"]


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "itemknncbf_tiny.npz"), allow_pickle=True)


@pytest.mark.parametrize("prefix", PREFIXES)
def test_oracle_equals_the_reference(gold, prefix):
    """kNN before the scatter, scores_matrix and full_sort_predict.  The kNN is the reference's expression in fp32 through
    the CPU's GEMM, whose low bits depend on the instruction set it picks: the restatement must give the recorded
    neighbours except near ties, with every value within the fp32 error bound of the exact similarity (bit-identical on
    the machine that recorded the file).  The sums are exact fp32 arithmetic of the recorded kNN values: bit for bit.  R's
    stored order is ascending on `tiny`, so the ascending-order sum (K9's contract) and the stored-order sum are the same
    sum, and both match."""
    from mmrec_b200.utils import synth
    G = lambda k: gold[prefix + k]
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    feats = KO.features(torch.from_numpy(np.asarray(v, np.float32)), torch.from_numpy(np.asarray(t, np.float32)))
    assert feats.shape == (i, 2 * f)
    shrink = int(G("cfg_shrink"))
    kv, ki = KO.item_sim_topk(feats, int(G("cfg_knn_k")), shrink)
    ok, _ = KO.knn_agrees(kv.numpy(), ki.numpy(), G("knn_val"), G("knn_ind"), feats, shrink)
    assert ok
    ok, _ = KO.knn_agrees(*(a.numpy() for a in KO.item_sim_topk_f64(feats, int(G("cfg_knn_k")), shrink)), G("knn_val"), G("knn_ind"),
                          feats, shrink)
    assert ok
    assert str(G("r_sum_order")) == "both" and bool(G("r_stored_ascending"))
    args = (G("inter_row"), G("inter_col"), G("inter_val"), int(G("n_users")), G("knn_val"), G("knn_ind"))
    for order in ("ascending", "stored"):
        sm = KO.ordered_scores(*args, order=order)
        assert np.array_equal(sm.view(np.uint32), G("scores_matrix").view(np.uint32)), order
    assert np.array_equal(sm[G("eval_users")].view(np.uint32), G("scores").view(np.uint32))


@pytest.mark.parametrize("prefix", PREFIXES)
def test_itemknncbf_class_against_the_reference(prefix):
    """The kNN graph (the stand-in evaluates the similarity in float64: the recorded neighbours except near ties, values
    within the fp32 bound), the predictions to 1e-6 relative, the one parameter, and the valid / test metrics of
    `Trainer.evaluate`."""
    r = run("itemknncbf_contract_worker.py", prefix)
    assert r["knn_ok"] and r["dummy_ok"] and r["params"] == ["dummy_embeddings"]
    assert r["score_err"] < 1e-6
    assert_metrics(r)


def _crafted_rows():
    """(dense row, masked items, k): few candidates, negative and -0.0 sums, masks over candidates and non-candidates,
    duplicates and out-of-range items in the mask, k beyond the unmasked count."""
    n = 40
    cases = []
    r = np.zeros(n, np.float32)
    r[[3, 17, 25]] = [0.5, 2.0, 0.5]
    cases += [(r, [], 10), (r, [17, 4, 4, 99, -1], 10), (r, [3, 17, 25], 5)]
    r = np.zeros(n, np.float32)
    r[[1, 2, 9, 30]] = [-1.0, 3.0, -0.25, 1.0]
    r[12] = -0.0
    cases += [(r, [], 40), (r, [2, 0], 40), (r, list(range(5, 40)), 40), (r, list(range(0, 38)), 10)]
    r = np.zeros(n, np.float32)
    r[[0, 39]] = [-0.0, -0.0]
    cases += [(r, [1], 40), (r, [], 1)]
    rng = np.random.default_rng(0)
    r = np.zeros(n, np.float32)
    c = rng.choice(n, 25, replace=False)
    r[c] = rng.standard_normal(25).astype(np.float32)
    r[c[:3]] = r[c[3]]                                                # equal values: ascending index
    cases += [(r, list(rng.choice(n, 8)), k) for k in (1, 7, 30, 40)]
    return cases


@pytest.mark.parametrize("case", range(len(_crafted_rows())))
def test_sparse_ranking_rule_equals_the_dense_ranking(case):
    row, masked, k = _crafted_rows()[case]
    cols = np.nonzero(row.view(np.uint32))[0]
    v, i = KO.sparse_rank(cols, row[cols], masked, len(row), k)
    dv, di = KO.dense_rank(row, masked, k)
    assert np.array_equal(i, di) and np.array_equal(v.view(np.uint32), dv.view(np.uint32))
    if not np.signbit(row[row == 0]).any():                           # without -0.0, float_key order is torch's order
        t = torch.from_numpy(row.copy())
        m = torch.tensor([x for x in masked if 0 <= x < len(row)], dtype=torch.int64)
        t[m] = -1e10
        tv, ti = torch.sort(t, descending=True, stable=True)
        assert np.array_equal(ti[:k].numpy(), i) and np.array_equal(tv[:k].numpy(), v)


def test_itemknncbf_config_keys():
    import yaml
    cfg = yaml.safe_load(open(os.path.join(ROOT, "mmrec_b200", "configs", "model", "ItemKNNCBF.yaml")))
    assert cfg["knn_k"] == [10] and cfg["shrink"] == [10] and cfg["req_training"] is False and cfg["epochs"] == 1
    assert sorted(cfg["hyper_parameters"]) == ["knn_k", "shrink"]


def test_new_entry_points_reject_bad_arguments_without_a_gpu():
    from mmrec_b200 import _lib, ops
    lib = _lib.load()
    X = 16                                                            # never dereferenced: the checks come first
    assert lib.mmrec_knn_topk_shrink_f32(10, X, 8, 8, 10, None, 11, X, 10.0, X, X, X, 1 << 20, None) == -1    # k > n
    assert lib.mmrec_knn_topk_shrink_f32(10, X, 8, 8, 10, None, 5, None, 10.0, X, X, X, 1 << 20, None) == -1  # null norms
    assert b"knn_topk" in lib.mmrec_last_error()
    assert lib.mmrec_sparse_scores_f32(-1, None, 10, X, X, X, X, X, X, X, 10, None) == -1
    assert lib.mmrec_sparse_scores_f32(4, None, 10, X, X, X, X, X, X, X, 5, None) == -1                  # ldo < n_items
    assert lib.mmrec_sparse_scores_f32(0, None, 10, None, None, None, None, None, None, None, 10, None) == 0
    assert b"sparse_scores" in lib.mmrec_last_error()
    top = lib.mmrec_sparse_score_topk_f32
    assert top(4, None, 10, X, X, X, X, X, X, 0, None, None, 11, X, X, X, 1 << 20, None) == -1           # k > n_items
    assert top(4, None, 10, X, X, X, X, X, X, 3, None, None, 5, X, X, X, 1 << 20, None) == -1            # null mask
    assert top(4, None, 10, X, X, X, X, X, X, 0, None, None, 5, X, X, X, 0, None) == -2                  # workspace too small
    assert b"sparse_score_topk" in lib.mmrec_last_error()
    assert lib.mmrec_sparse_score_topk_workspace_bytes(4096, 23000, 50000, 2048) == 0
    assert lib.mmrec_sparse_score_topk_workspace_bytes(4096, 23000, 50000, 50) > 0
    assert lib.mmrec_debug_sparse_topk_fallback_rows() == -1
    with pytest.raises(ops.MMRecError):
        ops.knn_topk(torch.zeros(4, 8), 2, shrink=10.0)
