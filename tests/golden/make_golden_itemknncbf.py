"""Generate ItemKNNCBF's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF (src/models/itemknncbf.py):

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_itemknncbf.py

Same harness and dataset (`tiny`: F = 128 per modality, 256 concatenated) as make_golden.py.  One file,
itemknncbf_tiny.npz, with every field twice: prefix `s10_` at the YAML's shrink = 10 and `s0_` at shrink = 0.  Per setting:
the train interactions in the order the model's COO holds them, the kNN values and indices before the scatter (recorded from
the reference's own `torch.topk` call inside `build_item_sim_matrix`), `scores_matrix`, `full_sort_predict` on the first
valid batch, and the valid / test metrics of the reference's Trainer.

The sum order of `torch.mm(r_matrix, item_sim)`: `r_sum_order` records which restatement of tests/itemknncbf_oracle.py
(`ordered_scores`, R's entries per user in ascending column order -- K9's order -- or in stored order) reproduces
`scores_matrix` bit for bit, and `r_stored_ascending` whether the stored order already is ascending.
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import itemknncbf_oracle as KO  # noqa: E402
import make_golden  # noqa: E402
import ref_loader  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512}
SHRINKS = {"s10_": 10, "s0_": 0}
OUT = "itemknncbf_tiny.npz"


def dump(shrink, prefix, g):
    from common.trainer import Trainer
    rec = {}
    topk = torch.topk

    def spy(*a, **kw):                                                # the first top-k of the model: its kNN graph
        out = topk(*a, **kw)
        if "val" not in rec:
            rec["val"], rec["ind"] = out[0].clone(), out[1].clone()
        return out
    torch.topk = spy
    try:
        config, train_data, valid_data, test_data, model = make_golden.build("ItemKNNCBF", dict(COMMON, shrink=[shrink]))
    finally:
        torch.topk = topk
    assert config["shrink"] == shrink and not config["req_training"]
    inter = train_data.inter_matrix(form="coo").astype(np.float32)
    g[prefix + "inter_row"], g[prefix + "inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
    g[prefix + "inter_val"] = inter.data.astype(np.float32)
    g[prefix + "n_users"], g[prefix + "n_items"] = np.int64(model.n_users), np.int64(model.n_items)
    g[prefix + "cfg_knn_k"], g[prefix + "cfg_shrink"] = np.float64(config["knn_k"]), np.float64(config["shrink"])
    g[prefix + "knn_val"], g[prefix + "knn_ind"] = rec["val"].numpy().copy(), rec["ind"].numpy().copy()
    sm = model.scores_matrix.numpy().copy()
    g[prefix + "scores_matrix"] = sm
    g[prefix + "dummy_embeddings"] = model.dummy_embeddings.detach().numpy().copy()
    # which order of R's non-zeros the reference sums in
    args = (inter.row, inter.col, inter.data, model.n_users, g[prefix + "knn_val"], g[prefix + "knn_ind"])
    asc = np.array_equal(KO.ordered_scores(*args, order="ascending").view(np.uint32), sm.view(np.uint32))
    sto = np.array_equal(KO.ordered_scores(*args, order="stored").view(np.uint32), sm.view(np.uint32))
    order = "both" if asc and sto else "ascending" if asc else "stored" if sto else "neither"
    g[prefix + "r_sum_order"] = np.array(order)
    g[prefix + "r_stored_ascending"] = np.bool_(bool(np.all(np.diff(inter.row * model.n_items + inter.col) > 0)))
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        scores = model.full_sort_predict(eb)
        g[prefix + "eval_users"], g[prefix + "eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        g[prefix + "scores"] = scores.numpy().copy()
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    test_res = trainer.evaluate(test_data, is_test=True)
    g[prefix + "metric_names"] = np.array(list(res.keys()))
    g[prefix + "metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g[prefix + "test_metric_values"] = np.array([test_res[k] for k in res], dtype=np.float64)
    print(f"ItemKNNCBF shrink={shrink}: R summed in {order} order (stored ascending: {bool(g[prefix + 'r_stored_ascending'])}), "
          f"valid {dict(zip(list(res)[:2], list(res.values())[:2]))}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    data_root = ref_loader.run_dir(tmp)
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    import logging
    logging.disable(logging.CRITICAL)
    g = {}
    for prefix, shrink in SHRINKS.items():
        dump(shrink, prefix, g)
    np.savez_compressed(os.path.join(HERE, OUT), **g)
    print(f"wrote {OUT} ({os.path.getsize(os.path.join(HERE, OUT)) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
