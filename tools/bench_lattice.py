"""LATTICE measurement at the baby, sports and clothing shapes (synthetic graphs of those sizes, image features F = 4096,
text features F = 384, B = 2048, lightgcn, knn_k 10, n_layers 1):

  * a graph-building training step (the first batch after `pre_epoch_processing`: the learned graph rebuilt under
    autograd) and an ordinary step (the stored graph, detached), each `calculate_loss` + backward + the Trainer's
    optimizer step;
  * one `Trainer.evaluate` on the validation split (the model builds the learned graph once per evaluation);
  * beside each, the reference's dense expressions on the device (`src/models/lattice.py:132-197`, `src/utils/utils.py:
    119-137`): `build_sim`, `build_knn_neighbourhood`, the weighted sums, `compute_normalized_laplacian` with `diagflat`
    products and `torch.mm(item_adj, h)` on [I, I] matrices, `torch.sparse.mm` for `norm_adj`; its evaluation rebuilds the
    graph for every evaluation batch, timed as one dense graph-building forward per batch plus the model's scoring.

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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lgmrec import card, timed  # noqa: E402


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
    config = Config("LATTICE", shape, {"data_path": data + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("LATTICE")(config, train).to(config["device"])
    return config, train, valid, model


class DenseReference:
    """The reference's forward on the device from the model's own parameters (lightgcn), dense [I, I] graphs."""

    def __init__(self, model):
        self.m = model
        r, c, v = model.norm_adj.coo()
        n = model.n_users + model.n_items
        self.norm_adj = torch.sparse_coo_tensor(torch.stack([r, c]), v, (n, n)).coalesce()
        self.image_original_adj = model.image_original_adj.to_dense()
        self.text_original_adj = model.text_original_adj.to_dense()
        self.item_adj = None

    @staticmethod
    def build_sim(context):
        cn = context.div(torch.norm(context, p=2, dim=-1, keepdim=True))
        return torch.mm(cn, cn.transpose(1, 0))

    @staticmethod
    def knn(adj, topk):
        val, ind = torch.topk(adj, topk, dim=-1)
        return torch.zeros_like(adj).scatter_(-1, ind, val)

    @staticmethod
    def laplacian(adj):
        d = torch.pow(torch.sum(adj, -1), -0.5)
        d[torch.isinf(d)] = 0.
        dm = torch.diagflat(d)
        return torch.mm(torch.mm(dm, adj), dm)

    def forward(self, build_item_graph):
        m = self.m
        image_feats = m.image_trs(m.image_embedding.weight)
        text_feats = m.text_trs(m.text_embedding.weight)
        if build_item_graph:
            w = m.softmax(m.modal_weight)
            learned = w[0] * self.knn(self.build_sim(image_feats), m.knn_k) + w[1] * self.knn(self.build_sim(text_feats), m.knn_k)
            original = w[0] * self.image_original_adj + w[1] * self.text_original_adj
            self.item_adj = None
            self.item_adj = (1 - m.lambda_coeff) * self.laplacian(learned) + m.lambda_coeff * original
        else:
            self.item_adj = self.item_adj.detach()
        h = m.item_id_embedding.weight
        for _ in range(m.n_layers):
            h = torch.mm(self.item_adj, h)
        ego = torch.cat((m.user_embedding.weight, m.item_id_embedding.weight), dim=0)
        embs = [ego]
        for _ in range(m.n_ui_layers):
            ego = torch.sparse.mm(self.norm_adj, ego)
            embs.append(ego)
        all_e = torch.stack(embs, dim=1).mean(dim=1)
        u_g, i_g = torch.split(all_e, [m.n_users, m.n_items], dim=0)
        return u_g, i_g + F.normalize(h, p=2, dim=1)

    def loss(self, batch, build):
        u_g, i_g = self.forward(build)
        mf, emb, reg = self.m.bpr_loss(u_g[batch[0]], i_g[batch[1]], i_g[batch[2]])
        return mf + emb + reg


def run_shape(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_lattice_")
    config, train, valid, model = build_model(shape, batch_size, tmp)
    trainer = Trainer(config, model)
    batch = next(iter(train)).to(config["device"])
    ref = DenseReference(model)
    opt = trainer.optimizer
    model.train()
    model.pre_epoch_processing()
    model.calculate_loss(batch)
    res = {"shape": shape, "users": model.n_users, "items": model.n_items, "norm_adj_nnz": model.norm_adj.nnz,
           "item_adj_nnz": model.item_adj.nnz, "batch": int(batch.shape[1]), "optimizer": type(opt).__name__,
           "dense_item_matrix_bytes": 4 * model.n_items ** 2}

    def step(loss_fn):
        opt.zero_grad()
        loss_fn().backward()
        opt.step()

    routes = {
        "build_step": lambda: step(lambda: (model.pre_epoch_processing(), model.calculate_loss(batch))[1]),
        "plain_step": lambda: step(lambda: model.calculate_loss(batch)),
        "build_step_ref": lambda: step(lambda: ref.loss(batch, True)),
        "plain_step_ref": lambda: step(lambda: ref.loss(batch, False)),
    }
    n_eval_batches = sum(1 for _ in valid)

    def eval_ref():
        with torch.no_grad():
            for _ in range(n_eval_batches):
                ref.forward(True)

    def evaluate():
        model.invalidate_eval_cache()
        trainer.evaluate(valid)
        model.train()
    routes["evaluate"] = evaluate
    routes["evaluate_ref_graphs"] = eval_ref
    order = ["build_step", "plain_step", "build_step_ref", "plain_step_ref", "evaluate", "evaluate_ref_graphs"]
    times = {k: [] for k in order}
    peaks = {}
    for name in order:                                                # warm-up and peak memory, one route at a time
        if name.startswith("plain"):
            routes[name.replace("plain", "build")]()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        routes[name]()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    for _ in range(reps):                                             # interleaved rounds
        for name in order:
            if name.startswith("plain"):
                routes[name.replace("plain", "build")]()
            times[name].append(timed(routes[name], 1)["median_s"])
    for name in order:
        t = sorted(times[name])
        res[name] = {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1], "peak_bytes_above_model": int(peaks[name])}
    res["eval_batches"] = n_eval_batches
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lattice needs a CUDA device")
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
