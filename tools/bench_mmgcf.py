"""MMGCF measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096, text
features F = 384, B = 2048, n_ui_layers 2, dropout 0.2), for `fusion_mode` / `weighting` mean / normalized and
concat / alpha:

  * one training step (`calculate_loss` + backward + `FusedAdam.step`), the routes interleaved rep by rep, with the peak
    memory of each above the model:
      (a) "step": the model as built -- K1 propagation, K2 on the 2B gathered rows, the fusion kernel on those rows;
      (b) "step_torch_fusion": the same model with the fusion as the reference's torch expression on the gathered rows
          (tests/golden/mmgcf_golden.torch_late_fuse; element-wise modes only: concat has no kernel, so (b) is (a));
      (c) "step_ref": the reference's expressions on the device (`src/models/mmgcf.py:124-142,256-284`): `torch.sparse.mm`
          layers and the stacked mean, full-table `F.linear` of both feature tables, the torch fusion of all items, then
          the gathers;
  * `pre_epoch_processing` (the pruning draw and the CSR rebuild);
  * one `Trainer.evaluate` on the validation split.

Each route's `loss` is taken before its warm-up steps, so later routes see a model the earlier ones have trained.  Device
events after a warm-up, median and range over `--reps`.  The card name, power limit and maximum SM clock are read
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from bench_lgmrec import card, timed  # noqa: E402
from mmgcf_golden import torch_late_fuse  # noqa: E402

MODES = (("mean", "normalized"), ("concat", "alpha"))


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def build_model(shape, batch_size, fusion, weighting, data):
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    config = Config("MMGCF", shape, {"data_path": data + "/", "train_batch_size": batch_size, "fusion_mode": [fusion],
                                     "weighting": [weighting], "n_ui_layers": [2], "dropout": [0.2]})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("MMGCF")(config, train).to(config["device"])
    return config, train, valid, model


def ref_loss(model, A, interaction):
    """Route (c): the reference's `calculate_loss` as its own expressions, on the device."""
    users, pos, neg = interaction[0], interaction[1], interaction[2]
    ego = torch.cat([model.user_embedding.weight, model.item_id_embedding.weight], dim=0)
    layers = [ego]
    for _ in range(model.n_ui_layers):
        ego = torch.sparse.mm(A, ego)
        layers.append(ego)
    ua, ia = torch.split(torch.stack(layers, dim=1).mean(dim=1), [model.n_users, model.n_items], dim=0)
    feats = [F.linear(model.image_embedding.weight, model.image_trs.weight, model.image_trs.bias),
             F.linear(model.text_embedding.weight, model.text_trs.weight, model.text_trs.bias)]
    if model.fusion_mode == "concat":
        ia = model._concat_fusion(ia, feats)
    else:
        alpha = torch.sigmoid(model.mm_alpha) if model.weighting == "alpha" else None
        ia = torch_late_fuse(ia, feats[0], feats[1], model.fusion_mode, model.weighting, alpha=alpha)
    mf = model.bpr_loss(ua[users], ia[pos], ia[neg])
    reg = (model.user_embedding.weight[users].norm(2).pow(2) + model.item_id_embedding.weight[pos].norm(2).pow(2)
           + model.item_id_embedding.weight[neg].norm(2).pow(2)) / (2 * len(users))
    return mf + model.reg_weight * reg


def run_mode(shape, data, reps, batch_size, fusion, weighting):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    config, train, valid, model = build_model(shape, batch_size, fusion, weighting, data)
    trainer = Trainer(config, model)
    torch.manual_seed(0)
    model.pre_epoch_processing()
    r, c, v = model.masked_adj.coo()
    A = torch.sparse_coo_tensor(torch.stack([r, c]), v, (model.n_nodes, model.n_nodes)).coalesce()
    batch0 = next(iter(train)).to(config["device"])
    res = {"fusion_mode": fusion, "weighting": weighting, "batch": int(batch0.shape[1]),
           "optimizer": type(trainer.optimizer).__name__}
    model.train()
    own_fuse = ops.late_fuse
    routes = {"step": (own_fuse, model.calculate_loss)}
    if fusion != "concat":
        routes["step_torch_fusion"] = (torch_late_fuse, model.calculate_loss)
    routes["step_ref"] = (own_fuse, lambda b: ref_loss(model, A, b))

    def use(name):
        ops.late_fuse = routes[name][0]
        return routes[name][1]

    def step(loss_fn):
        trainer.optimizer.zero_grad()
        loss_fn(batch0).backward()
        trainer.optimizer.step()

    peak, losses = {}, {}
    try:
        for name in routes:
            fn = use(name)
            with torch.no_grad():
                losses[name] = float(fn(batch0))
            for _ in range(3):
                step(fn)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            step(fn)
            torch.cuda.synchronize()
            peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        ts = {k: [] for k in routes}
        for _ in range(reps):
            for name in routes:
                fn = use(name)
                ts[name].append(timed(lambda: step(fn), 1)["median_s"])
    finally:
        ops.late_fuse = own_fuse
    for name in routes:
        res[name] = dict(_summary(ts[name]), peak_mib=peak[name], loss=losses[name])
    if "step_torch_fusion" in res:
        res["speedup_vs_torch_fusion"] = res["step_torch_fusion"]["median_s"] / res["step"]["median_s"]
    res["speedup_vs_ref"] = res["step_ref"]["median_s"] / res["step"]["median_s"]
    pe = []
    for _ in range(max(3, reps // 3)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.pre_epoch_processing()
        torch.cuda.synchronize()
        pe.append(time.perf_counter() - t0)
    res["pre_epoch_processing"] = _summary(pe)
    model.eval()
    trainer.evaluate(valid)
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(3, reps // 3))
    return res


def run_shape(shape, reps, batch_size, modes):
    from mmrec_b200.utils import synth
    u, i, e, d, _ = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    rng = np.random.default_rng(1)
    data = os.path.join(tempfile.mkdtemp(prefix="mmrec_bench_mmgcf_"), "data")
    synth.write_dataset(data, shape, gr, rng.standard_normal((i, 4096), dtype=np.float32), rng.standard_normal((i, 384), dtype=np.float32))
    return {"shape": shape, "users": u, "items": i, "F_image": 4096, "F_text": 384,
            "modes": [run_mode(shape, data, reps, batch_size, f, w) for f, w in modes]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--modes", default=",".join(f"{f}/{w}" for f, w in MODES))
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    modes = [tuple(m.split("/")) for m in a.modes.split(",")]
    out = {"card": card(), "shapes": [run_shape(sh, a.reps, a.batch, modes) for sh in a.shapes.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
