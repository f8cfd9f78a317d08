"""DualGNN measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096,
text features F = 384, B = 2048, `aggr_mode: add`):

  * one training step (`calculate_loss` + backward + `FusedAdam.step`), three routes interleaved rep by rep, with the
    peak memory of each:
      (a) "step": the model as built -- both towers as one width-128 K1 propagation, the user graph as K1 on the epoch's CSR;
      (b) "step_ref_user_graph": the same model with the reference's user-graph expression (`User_Graph_sample`,
          `src/models/dualgnn.py:259-266`): the epoch's index as a Python list of lists, `features[index]` (a [U, 40, 64]
          gather, the list converted every batch), a batched matmul, then `user_rep +`;
      (c) "step_ref": the reference's expressions restated here on the device: each tower's two convs as PyG's 'add'
          message passing (gather x[row], scale by the gcn norm, `index_add` at col), `MLP` as `F.linear`, and (b)'s user
          graph;
  * `pre_epoch_processing` (host sample + the user-graph CSR and its transpose);
  * one `Trainer.evaluate` on the validation split;
  * the host build of `synth.write_user_graph_dict` at each shape (once).

Device events after a warm-up, median and range over `--reps`.  The card name, power limit and maximum SM clock are read
(read-only) in the same run.  Prints JSON; writes it to --out only when given."""
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

from bench_lgmrec import card, timed  # noqa: E402


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def ref_user_graph(model):
    """Route (b)'s `User_Graph_sample.forward` plus `user_rep + h_u1`, on the epoch's index kept as the reference keeps it."""
    index = model.epoch_user_graph.tolist()

    def forward(features, user_graph, user_matrix=None, base=None):
        u_features = features[index]
        u_pre = torch.matmul(model.user_weight_matrix.unsqueeze(1), u_features).squeeze()
        return u_pre if base is None else base + u_pre
    return forward


def ref_propagate_sum(edge_index, n_nodes):
    """Route (c)'s towers: PyG's 'add' conv (`dualgnn.py:325-341` under PyG's scatter) twice per 64-wide tower."""
    ei = edge_index[:, edge_index[0] != edge_index[1]]
    row, col = ei[0], ei[1]

    def conv(x):
        deg = torch.zeros(n_nodes, dtype=x.dtype, device=x.device).index_add_(0, row, torch.ones_like(row, dtype=x.dtype))
        dis = deg.pow(-0.5)
        msg = (dis[row] * dis[col]).view(-1, 1) * x.index_select(0, row)
        return torch.zeros(n_nodes, x.shape[1], dtype=x.dtype, device=x.device).index_add_(0, col, msg)

    def prop(A, x, n_layers):
        outs = []
        for k in range(x.shape[1] // 64):
            xk = x[:, 64 * k:64 * (k + 1)]
            h = conv(xk)
            outs.append(h + xk + conv(h))
        return torch.cat(outs, dim=1) if len(outs) > 1 else outs[0]
    return prop


def build_model(shape, batch_size, tmp):
    from mmrec_b200.utils import synth
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    u, i, e, d, _ = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    rng = np.random.default_rng(1)
    v = rng.standard_normal((i, 4096), dtype=np.float32)
    t = rng.standard_normal((i, 384), dtype=np.float32)
    data = os.path.join(tmp, "data")
    synth.write_dataset(data, shape, gr, v, t)
    t0 = time.perf_counter()
    synth.write_user_graph_dict(data, shape, gr)
    host_build_s = time.perf_counter() - t0
    config = Config("DualGNN", shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("DualGNN")(config, train).to(config["device"])
    return config, train, valid, model, host_build_s


def run_shape(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_dualgnn_")
    config, train, valid, model, host_build_s = build_model(shape, batch_size, tmp)
    trainer = Trainer(config, model)
    np.random.seed(0)
    model.pre_epoch_processing()
    batch0 = next(iter(train)).to(config["device"])
    res = {"shape": shape, "users": model.n_users, "items": model.n_items, "adj_nnz": model.adj.nnz,
           "user_graph_nnz": model.user_graph_csr.nnz, "F_image": int(model.v_feat.shape[1]), "F_text": int(model.t_feat.shape[1]),
           "batch": int(batch0.shape[1]), "optimizer": type(trainer.optimizer).__name__,
           "write_user_graph_dict_s": host_build_s}
    model.train()
    own = {"propagate_sum": ops.propagate_sum, "project": ops.project}
    ref_graph = ref_user_graph(model)
    ref_prop = ref_propagate_sum(model.edge_index, model.n_users + model.n_items)

    def ref_project(table, weight, bias=None, idx=None, l2_normalize=False):
        return F.linear(table, weight, bias)

    routes = {"step": (own["propagate_sum"], own["project"], None),
              "step_ref_user_graph": (own["propagate_sum"], own["project"], ref_graph),
              "step_ref": (ref_prop, ref_project, ref_graph)}

    def use(name):
        prop, proj, ug = routes[name]
        ops.propagate_sum, ops.project = prop, proj
        if ug is None:
            model.user_graph.__dict__.pop("forward", None)
        else:
            model.user_graph.forward = ug

    def step():
        trainer.optimizer.zero_grad()
        model.calculate_loss(batch0.clone()).backward()              # forward offsets the item ids in place
        trainer.optimizer.step()

    peak, losses = {}, {}
    try:
        for name in routes:
            use(name)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step()
            torch.cuda.synchronize()
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
        res[name] = dict(_summary(ts[name]), peak_mib=peak[name], loss_after_steps=losses[name])
    res["speedup_vs_ref_user_graph"] = res["step_ref_user_graph"]["median_s"] / res["step"]["median_s"]
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
    ap.add_argument("--reps", type=int, default=20)
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
