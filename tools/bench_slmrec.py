"""SLMRec measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, d = 64, layer_num = 3, the
`pre` adjacency):

  * the propagation alone, forward + backward (a fixed upstream gradient), three routes interleaved rep by rep:
      (a) "wide":  one `ops.propagate_mean` of the [N, 3d] ego table -- K1 at width 3d, what the model runs;
      (b) "three": three `ops.propagate_mean` of the [N, d] views -- K1 at width d, three times;
      (c) "torch": the reference's `compute_graph` x 3 on the device (`torch.sparse.mm` per layer, stack, mean; autograd);
    the three outputs are compared (wide against three: bit equality; against torch: max relative difference);
  * one full training step of the model class (`calculate_loss` + backward + `FusedAdam.step`, B = 2048), as built and with
    its propagation swapped for route (b), interleaved, with the peak memory of each;
  * one `Trainer.evaluate` on the validation split.

Device events after a warm-up, median and range over `--reps`.  The card name, power limit and maximum SM clock are read
(read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lgmrec import card, timed  # noqa: E402


def _summary(ts):
    t = sorted(ts)
    return {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}


def three_views(A, ego, L, _propagate=None):
    """Route (b): the three d-wide propagations, concatenated."""
    from mmrec_b200 import ops
    prop = _propagate or ops.propagate_mean
    d = ego.shape[1] // 3
    return torch.cat([prop(A, ego[:, k * d:(k + 1) * d], L) for k in range(3)], dim=1)


def propagation(shape, reps, L=3):
    from mmrec_b200 import graph, ops
    from mmrec_b200.utils import synth
    u, i, e, d, _ = synth.SHAPES[shape]
    g = synth.make_graph(u, i, e, seed=0).split(0)
    A = graph.build_slmrec_adj((g[0], g[1]), u, i, "cuda", "pre")
    r, c, v = A.coo()
    T = torch.sparse_coo_tensor(torch.stack((r, c)), v, (A.n_rows, A.n_cols)).coalesce()
    gen = torch.Generator(device="cuda").manual_seed(0)
    ego0 = torch.randn(A.n_rows, 3 * d, device="cuda", generator=gen) * 0.1
    up = torch.randn(A.n_rows, 3 * d, device="cuda", generator=gen)

    def torch_route(ego):
        outs = []
        for k in range(3):
            x = ego[:, k * d:(k + 1) * d]
            layers = [x]
            for _ in range(L):
                x = torch.sparse.mm(T, x)
                layers.append(x)
            outs.append(torch.stack(layers, dim=1).mean(dim=1))
        return torch.cat(outs, dim=1)

    routes = {"wide": lambda x: ops.propagate_mean(A, x, L), "three": lambda x: three_views(A, x, L), "torch": torch_route}

    def run(route):
        ego = ego0.clone().requires_grad_(True)
        out = routes[route](ego)
        out.backward(up)
        return out.detach(), ego.grad

    res = {"shape": shape, "n_nodes": A.n_rows, "nnz": A.nnz, "d": d, "width": 3 * d, "layers": L}
    got = {k: run(k) for k in routes}
    res["wide_equals_three"] = {"forward": bool(torch.equal(got["wide"][0], got["three"][0])),
                                "backward": bool(torch.equal(got["wide"][1], got["three"][1]))}
    res["max_rel_vs_torch"] = {k: [float(((got[k][j] - got["torch"][j]).abs().max() / got["torch"][j].abs().max()).item()) for j in (0, 1)]
                               for k in ("wide", "three")}
    for k in routes:
        for _ in range(3):
            run(k)
    ts = {k: [] for k in routes}
    for _ in range(reps):
        for k in routes:
            ts[k].append(timed(lambda: run(k), 1)["median_s"])
    for k in routes:
        res[k] = _summary(ts[k])
    res["speedup_wide_vs_three"] = res["three"]["median_s"] / res["wide"]["median_s"]
    res["speedup_wide_vs_torch"] = res["torch"]["median_s"] / res["wide"]["median_s"]
    return res


def train_and_eval(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.utils import synth
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_slmrec_")
    u, i, e, d, f = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), shape, gr, v, t)
    config = Config("SLMRec", shape, {"data_path": os.path.join(tmp, "data") + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("SLMRec")(config, train).to(config["device"])
    trainer = Trainer(config, model)
    batch = next(iter(train)).to(config["device"])
    model.train()
    wide = ops.propagate_mean

    def step():
        trainer.optimizer.zero_grad()
        model.calculate_loss(batch).backward()
        trainer.optimizer.step()

    res = {"shape": shape, "users": u, "items": i, "edges": e, "F": f, "batch": int(batch.shape[1]),
           "optimizer": type(trainer.optimizer).__name__}
    routes = {"step": wide, "step_three_views": lambda A, ego, L: three_views(A, ego, L, wide)}
    peak = {}
    for name, fn in routes.items():
        ops.propagate_mean = fn
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step()
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    ts = {k: [] for k in routes}
    try:
        for _ in range(reps):
            for name, fn in routes.items():
                ops.propagate_mean = fn
                ts[name].append(timed(step, 1)["median_s"])
    finally:
        ops.propagate_mean = wide
    for name in routes:
        res[name] = dict(_summary(ts[name]), peak_mib=peak[name])
    res["step_speedup_wide_vs_three"] = res["step_three_views"]["median_s"] / res["step"]["median_s"]
    model.eval()
    trainer.evaluate(valid)
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(3, reps // 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    shapes = a.shapes.split(",")
    out = {"card": card(), "propagation": [propagation(sh, a.reps) for sh in shapes]}
    if not a.skip_train:
        out["train"] = [train_and_eval(sh, a.reps, a.batch) for sh in shapes]
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
