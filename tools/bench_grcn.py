"""GRCN measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096,
text features F = 384, B = 2048, n_layers 3, both modalities):

  (a) the model's training step (`calculate_loss` + backward + the Trainer's optimizer step) and one `Trainer.evaluate` on
      the validation split;
  (b) the same step with the edge attention taken through a composition of existing ops instead of the row kernel
      (`compose_attention` of tests/test_gpu_grcn.py: `sddmm` scores, `segment_reduce` max, width-1 K1 row sums,
      `spmm_values`);
  (c) the reference's expressions on the device (`reference_loss` of tests/test_gpu_grcn.py: PyG's message passing as
      `index_select` gathers of x_i / x_j, [2E, d] messages and `index_add_` scatters, the grouped softmax, the routing
      loop) with the same optimizer step;
plus the attention alone (forward + backward at d = 64 on the model's graph) by the kernel and by the composition.

Device events; each route warmed up first; median [min - max] over `--reps` rounds, the routes interleaved; peak memory
above the model for each.  The card name, power limit and maximum SM clock are read (read-only) in the same run.  Prints
JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from bench_lgmrec import card, timed  # noqa: E402
from test_gpu_grcn import compose_attention, reference_loss  # noqa: E402


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
    config = Config("GRCN", shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("GRCN")(config, train).to(config["device"])
    return config, train, valid, model


def run_shape(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_grcn_")
    config, train, valid, model = build_model(shape, batch_size, tmp)
    trainer = Trainer(config, model)
    batch = next(iter(train)).to(config["device"])
    opt = trainer.optimizer
    A = model.attn_adj
    deg = A.rowptr[1:] - A.rowptr[:-1]
    res = {"shape": shape, "users": model.n_users, "items": model.n_items, "attention_nnz": A.nnz, "batch": int(batch.shape[1]),
           "longest_row": int(deg.max()), "heavy_rows": int(ops.edge_attention_heavy_rows(A).numel()),
           "optimizer": type(opt).__name__}
    kernel_attention = ops.edge_attention
    model.train()

    def step(loss_fn):
        opt.zero_grad()
        loss_fn().sum().backward()
        opt.step()

    def composed_step():
        ops.edge_attention = compose_attention
        try:
            step(lambda: model.calculate_loss(batch))
        finally:
            ops.edge_attention = kernel_attention

    def evaluate():
        trainer.evaluate(valid)
        model.train()

    g = torch.Generator(device="cpu").manual_seed(0)
    X0 = torch.nn.functional.normalize(torch.randn(A.n_rows, 64, generator=g)).to(config["device"])
    uY = torch.randn(A.n_rows, 64, generator=g).to(config["device"])
    ua = torch.randn(A.nnz, generator=g).to(config["device"])

    def attention(fn):
        X = X0.clone().requires_grad_(True)
        Y, alpha = fn(A, X, X)
        torch.autograd.grad((Y * uY).sum() + (alpha * ua).sum(), (X,))

    routes = {"step": lambda: step(lambda: model.calculate_loss(batch)), "step_composed": composed_step,
              "step_ref": lambda: step(lambda: reference_loss(model, batch)), "evaluate": evaluate,
              "attention_kernel": lambda: attention(kernel_attention), "attention_composed": lambda: attention(compose_attention)}
    order = list(routes)
    times = {k: [] for k in order}
    peaks = {}
    for name in order:                                                # warm-up and peak memory, one route at a time
        routes[name]()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        routes[name]()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    for _ in range(reps):                                             # interleaved rounds
        for name in order:
            times[name].append(timed(routes[name], 1)["median_s"])
    for name in order:
        t = sorted(times[name])
        res[name] = {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1], "peak_bytes_above_model": int(peaks[name])}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grcn needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"card": card(), "results": [run_shape(s, a.reps, a.batch) for s in a.shapes.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
