"""DRAGON measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096,
text features F = 384, B = 2048, 'add', n_mm_layers 1, knn_k 10):

  * one training step (`calculate_loss` + backward + `FusedAdam.step`), the routes interleaved rep by rep, with the peak
    memory of each above the model and the library kernels it launches:
      (a) "step": the model as built -- the towers on K1 / K2, the torch weighting, `ops.spmm` on the user graph and on
          `mm_adj`;
      (c) "step_ref": the reference's expressions on the device: PyG-style gather / `index_add` convs for the towers and
          `F.linear` for `MLP` (tools/bench_dualgnn.py), the list-indexed [U, 40, 128] user-graph gather and batched
          matmul, and `torch.sparse.mm` for `mm_adj`;
  * `pre_epoch_processing` (host sample + the user-graph CSR and its transpose);
  * one `Trainer.evaluate` on the validation split.

Device events; each route warmed up first; median [min - max] over `--reps` interleaved rounds.  The card name, power limit
and maximum SM clock are read (read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_dualgnn import ref_propagate_sum, ref_user_graph  # noqa: E402
from bench_lgmrec import card, timed  # noqa: E402


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def build_model(shape, batch_size, tmp):
    from mmrec_b200.utils import synth
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    u, i, e, d, _ = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    rng = np.random.default_rng(1)
    data = os.path.join(tmp, "data")
    synth.write_dataset(data, shape, gr, rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32))
    synth.write_user_graph_dict(data, shape, gr)
    config = Config("DRAGON", shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("DRAGON")(config, train).to(config["device"])
    return config, train, valid, model


def run_shape(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_dragon_")
    config, train, valid, model = build_model(shape, batch_size, tmp)
    trainer = Trainer(config, model)
    np.random.seed(0)
    model.pre_epoch_processing()
    batch0 = next(iter(train)).to(config["device"])
    r, c, v = model.mm_adj.coo()
    M_sparse = torch.sparse_coo_tensor(torch.stack([r, c]), v, (model.n_items, model.n_items)).coalesce()
    res = {"shape": shape, "users": model.n_users, "items": model.n_items, "adj_nnz": model.adj.nnz,
           "user_graph_nnz": model.user_graph_csr.nnz, "mm_adj_nnz": model.mm_adj.nnz, "F_image": int(model.v_feat.shape[1]),
           "F_text": int(model.t_feat.shape[1]), "batch": int(batch0.shape[1]), "optimizer": type(trainer.optimizer).__name__}
    model.train()
    own = {"propagate_sum": ops.propagate_sum, "project": ops.project, "spmm": ops.spmm}
    ref_prop = ref_propagate_sum(model.edge_index, model.n_users + model.n_items)
    ref_graph = ref_user_graph(model)

    def ref_project(table, weight, bias=None, idx=None, l2_normalize=False):
        return F.linear(table, weight, bias)

    def ref_spmm(A, X, base=None):                                   # mm_adj: torch.sparse.mm (dragon.py:249-253)
        if A is not model.mm_adj:
            return own["spmm"](A, X, base=base)
        h = torch.sparse.mm(M_sparse, X)
        return h if base is None else base + h

    routes = {"step": (own["propagate_sum"], own["project"], own["spmm"], None),
              "step_ref": (ref_prop, ref_project, ref_spmm, ref_graph)}

    def use(name):
        ops.propagate_sum, ops.project, ops.spmm, ug = routes[name]
        if ug is None:
            model.user_graph.__dict__.pop("forward", None)
        else:
            model.user_graph.forward = ug

    def step():
        trainer.optimizer.zero_grad()
        model.calculate_loss(batch0.clone()).backward()              # forward offsets the item ids in place
        trainer.optimizer.step()

    peak, losses, launches = {}, {}, {}
    try:
        for name in routes:
            use(name)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            n0 = ops.launch_count()
            step()
            torch.cuda.synchronize()
            launches[name] = ops.launch_count() - n0
            peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            with torch.no_grad():
                losses[name] = float(model.calculate_loss(batch0.clone()))
        ts = {k: [] for k in routes}
        for _ in range(reps):
            for name in routes:
                use(name)
                ts[name].append(timed(step, 1)["median_s"])
    finally:
        use("step")
    for name in routes:
        res[name] = dict(_summary(ts[name]), peak_mib=peak[name], library_launches=launches[name], loss_after_steps=losses[name])
    res["speedup_vs_ref"] = res["step_ref"]["median_s"] / res["step"]["median_s"]
    pe = []
    for _ in range(max(3, reps // 4)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.pre_epoch_processing()
        torch.cuda.synchronize()
        pe.append(time.perf_counter() - t0)
    res["pre_epoch_processing"] = _summary(pe)
    step()
    model.eval()
    trainer.evaluate(valid)
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(3, reps // 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"card": card(), "shapes": [run_shape(sh, a.reps, a.batch) for sh in a.shapes.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
