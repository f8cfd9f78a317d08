"""PGL measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096, text
features F = 384; B = 2048; PGL's shipped configuration, dropout 0.2 and reg_weight 0, and reg_weight 0.1 as well):

  * one training step (`calculate_loss` + backward + `FusedAdam.step`), the routes interleaved rep by rep, with the peak
    memory of each above the model:
      (a) "step": the model as built -- `ops.pgl_loss` (one row kernel each way, K8 for the B x B sums);
      (b) "step_torch_loss": the same forward, the same four mask draws, and the loss as the reference's torch expression
          on the gathered rows (tests/golden/pgl_golden.torch_pgl_loss): isolates the loss kernel;
      (c) "step_ref": the reference's expressions on the device (`src/models/pgl.py:204-259`): F.linear + F.normalize of
          the feature tables, torch.sparse.mm for the sub-graph and the item graph, its bpr_loss, four nn.Dropout calls
          and its InfoNCE with the [B, B] matrices;
  * one `Trainer.evaluate` on the validation split.

Device events after a warm-up, median and range over `--reps`.  The card name, power limit and maximum SM clock are read
(read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from bench_lgmrec import card, timed  # noqa: E402
from pgl_golden import device_drop, info_nce, torch_pgl_loss  # noqa: E402


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def build_model(shape, batch_size, data, reg_weight):
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    config = Config("PGL", shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    config["reg_weight"] = reg_weight
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("PGL")(config, train).to(config["device"])
    return config, train, valid, model


def torch_sparse(A):
    r, c, v = A.coo()
    return torch.sparse_coo_tensor(torch.stack([r.long(), c.long()]), v, (A.n_rows, A.n_cols)).coalesce()


def ref_loss(model, interaction, sub, mm):
    """Route (c): the reference's `forward` + `calculate_loss` as its own expressions, on the device."""
    image_feats = F.normalize(F.linear(model.image_embedding.weight, model.image_trs.weight, model.image_trs.bias))
    text_feats = F.normalize(F.linear(model.text_embedding.weight, model.text_trs.weight, model.text_trs.bias))
    user_embeds = torch.cat([model.user_image.weight, model.user_text.weight], dim=1)
    item_embeds = torch.cat([image_feats, text_feats], dim=1)
    h = item_embeds
    for _ in range(model.n_layers):
        h = torch.sparse.mm(mm, h)
    ego = torch.cat((user_embeds, item_embeds), dim=0)
    all_e = [ego]
    for _ in range(model.n_ui_layers):
        ego = torch.sparse.mm(sub, ego)
        all_e.append(ego)
    all_e = torch.stack(all_e, dim=1).mean(dim=1)
    ua, ia = torch.split(all_e, [model.n_users, model.n_items], dim=0)
    ia = ia + h
    u, p, n = ua[interaction[0]], ia[interaction[1]], ia[interaction[2]]
    mf = -torch.mean(F.logsigmoid(torch.sum(torch.mul(u, p), dim=1) - torch.sum(torch.mul(u, n), dim=1)))
    cl = (info_nce(model.dropoutf(u), model.dropoutf(u)) + info_nce(model.dropoutf(p), model.dropoutf(p))) / 2
    return mf + model.reg_weight * cl


def run_model(shape, data, reps, batch_size, reg_weight):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    config, train, valid, model = build_model(shape, batch_size, data, reg_weight)
    trainer = Trainer(config, model)
    batch0 = next(iter(train)).to(config["device"])
    model.pre_epoch_processing()
    sub, mm = torch_sparse(model.sub_graph), torch_sparse(model.mm_adj)
    res = {"reg_weight": reg_weight, "dropout": float(model.dropoutf.p), "batch": int(batch0.shape[1]),
           "optimizer": type(trainer.optimizer).__name__, "sub_graph_nnz": int(model.sub_graph.nnz)}
    model.train()
    own = ops.pgl_loss

    def torch_loss(UA, IA, users, pos, neg, masks, p, rw):
        return torch_pgl_loss(UA, IA, users, pos, neg, masks, p, rw, drop=device_drop)
    routes = {"step": (own, model.calculate_loss), "step_torch_loss": (torch_loss, model.calculate_loss),
              "step_ref": (own, lambda b: ref_loss(model, b, sub, mm))}

    def use(route):
        ops.pgl_loss = routes[route][0]
        return routes[route][1]

    def step(loss_fn):
        trainer.optimizer.zero_grad()
        loss_fn(batch0).backward()
        trainer.optimizer.step()

    peak, losses = {}, {}
    try:
        for route in routes:
            fn = use(route)
            with torch.no_grad():
                losses[route] = float(fn(batch0))
            for _ in range(3):
                step(fn)
            trainer.optimizer.zero_grad(set_to_none=True)      # no route's stale gradients in the base
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step(fn)
            torch.cuda.synchronize()
            peak[route] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ts = {k: [] for k in routes}
        for _ in range(reps):
            for route in routes:
                fn = use(route)
                ts[route].append(timed(lambda: step(fn), 1)["median_s"])
    finally:
        ops.pgl_loss = own
    for route in routes:
        res[route] = dict(_summary(ts[route]), peak_mib=peak[route], loss=losses[route])
    res["speedup_vs_torch_loss"] = res["step_torch_loss"]["median_s"] / res["step"]["median_s"]
    res["speedup_vs_ref"] = res["step_ref"]["median_s"] / res["step"]["median_s"]
    model.eval()
    trainer.evaluate(valid)
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(3, reps // 3))
    return res


def run_shape(shape, reps, batch_size, reg_weights):
    from mmrec_b200.utils import synth
    u, i, e, d, _ = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    rng = np.random.default_rng(1)
    data = os.path.join(tempfile.mkdtemp(prefix="mmrec_bench_pgl_"), "data")
    synth.write_dataset(data, shape, gr, rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32))
    return {"shape": shape, "users": u, "items": i, "F_image": 4096, "F_text": 384,
            "runs": [run_model(shape, data, reps, batch_size, rw) for rw in reg_weights]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--reg-weights", default="0,0.1")
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rws = [float(x) for x in a.reg_weights.split(",")]
    out = {"card": card(), "shapes": [run_shape(sh, a.reps, a.batch, rws) for sh in a.shapes.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
