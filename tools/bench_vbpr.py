"""VBPR and BPR measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features
F = 4096, text features F = 384, so VBPR's raw table is 4480 wide; B = 2048):

  * one training step (`calculate_loss` + backward + `FusedAdam.step`), the routes interleaved rep by rep, with the peak
    memory of each above the model:
      (a) "step": the model as built -- VBPR's K2 on the 2B gathered rows, then `ops.bpr_mf_loss` (one kernel each way);
      (b) "step_torch_loss": the same gathered route with the loss as the reference's torch expression on the gathered
          rows (tests/golden/vbpr_golden.torch_bpr_mf_loss): isolates the loss kernel;
      (c) "step_ref": the reference's expressions on the device (`src/models/vbpr.py:69-98`, `bpr.py:62-86`): VBPR's
          full-table `F.linear` of the raw table and `torch.cat` with the ID table, then the gathers and the torch loss;
  * one `Trainer.evaluate` on the validation split.

Each route's `loss` is taken before its warm-up steps, so later routes see a model the earlier ones have trained.  Device
events after a warm-up, median and range over `--reps`.  The card name, power limit and maximum SM clock are read
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
from vbpr_golden import torch_bpr_mf_loss  # noqa: E402

MODELS = ("BPR", "VBPR")


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def build_model(name, shape, batch_size, data):
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    config = Config(name, shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model(name)(config, train).to(config["device"])
    return config, train, valid, model


def ref_loss(model, interaction):
    """Route (c): the reference's `forward` + `calculate_loss` as its own expressions, on the device."""
    if hasattr(model, "item_linear"):
        user_embeddings = model.u_embedding
        item_embeddings = torch.cat((model.i_embedding, F.linear(model.item_raw_features, model.item_linear.weight,
                                                                 model.item_linear.bias)), -1)
    else:
        user_embeddings, item_embeddings = model.user_embedding.weight, model.item_embedding.weight
    user_e = user_embeddings[interaction[0], :]
    pos_e, neg_e = item_embeddings[interaction[1], :], item_embeddings[interaction[2], :]
    pos_item_score, neg_item_score = torch.mul(user_e, pos_e).sum(dim=1), torch.mul(user_e, neg_e).sum(dim=1)
    return model.loss(pos_item_score, neg_item_score) + model.reg_weight * model.reg_loss(user_e, pos_e, neg_e)


def run_model(name, shape, data, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    config, train, valid, model = build_model(name, shape, batch_size, data)
    trainer = Trainer(config, model)
    batch0 = next(iter(train)).to(config["device"])
    res = {"model": name, "batch": int(batch0.shape[1]), "optimizer": type(trainer.optimizer).__name__,
           "raw_features": int(model.item_raw_features.shape[1]) if name == "VBPR" else 0}
    model.train()
    own = ops.bpr_mf_loss
    routes = {"step": (own, model.calculate_loss), "step_torch_loss": (torch_bpr_mf_loss, model.calculate_loss),
              "step_ref": (own, lambda b: ref_loss(model, b))}

    def use(route):
        ops.bpr_mf_loss = routes[route][0]
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
        ops.bpr_mf_loss = own
    for route in routes:
        res[route] = dict(_summary(ts[route]), peak_mib=peak[route], loss=losses[route])
    res["speedup_vs_torch_loss"] = res["step_torch_loss"]["median_s"] / res["step"]["median_s"]
    res["speedup_vs_ref"] = res["step_ref"]["median_s"] / res["step"]["median_s"]
    model.eval()
    trainer.evaluate(valid)
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(3, reps // 3))
    return res


def run_shape(shape, reps, batch_size, models):
    from mmrec_b200.utils import synth
    u, i, e, d, _ = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    rng = np.random.default_rng(1)
    data = os.path.join(tempfile.mkdtemp(prefix="mmrec_bench_vbpr_"), "data")
    synth.write_dataset(data, shape, gr, rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32))
    return {"shape": shape, "users": u, "items": i, "F_image": 4096, "F_text": 384,
            "models": [run_model(m, shape, data, reps, batch_size) for m in models]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"card": card(), "shapes": [run_shape(sh, a.reps, a.batch, a.models.split(",")) for sh in a.shapes.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
