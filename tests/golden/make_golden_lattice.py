"""Generate LATTICE's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_lattice.py

The unmodified model class (`src/models/lattice.py`) runs under `ref_loader.install()` (its `.cuda()` is the identity on
the CPU) with the harness, dataset and fields of make_golden.py and `train_batch_size` 512.  Each model is built in a
fresh data directory, so the constructor builds `image_adj_{k}.pt` / `text_adj_{k}.pt` instead of loading ones left by
another run.

Recorded (lattice_tiny.npz), per case: the SHA-256 of every initial `state_dict` entry and the parameter order; `norm_adj`
(indices and values); both original graphs; every [I, I] graph as its nonzero entries; on the graph-building batch (the first after
`pre_epoch_processing`) the learned `item_adj`, `forward`'s user and item embeddings, the loss and every gradient; on the
next batch (the stored graph, detached) the loss and every gradient; then in evaluation `full_sort_predict` of the first
validation batch, the trainer's top-50 of it and the validation and test metrics.  The `item_adj` evaluation leaves behind
is the graph-building batch's bit for bit (no optimizer step in between; asserted here), so it is not recorded twice.
Tensors of more than 4096 elements are kept as digest and sketch (`golden_io.put`), indices as int32 (the top-50
as int16).  To keep the file small, `forward`'s embeddings and the ordinary batch's gradients are recorded for the first
case only (the others record that batch's loss), and a case's learned graph only where it differs from the first case's
(lightgcn at two layers and mf draw the same initial weights, so they build the same graph).
Cases: lightgcn at n_layers 1 (no prefix) and 2 (`l2.`), `mf.`, `ngcf.` with mess_dropout 0, image only (`image.`) and
text only (`text.`).
traj_lattice_tiny.npz: two epochs of the reference's Trainer (lightgcn, both modalities) with its batches, losses and
metrics."""
import os
import random
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_io as G  # noqa: E402
import make_golden  # noqa: E402
import ref_loader  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512}
# prefix -> (config overrides, modalities)
CASES = {"": ({}, "vt"), "l2.": ({"n_layers": 2}, "vt"), "mf.": ({"cf_model": "mf"}, "vt"),
         "ngcf.": ({"cf_model": "ngcf", "mess_dropout": [0.0, 0.0]}, "vt"), "image.": ({}, "v"), "text.": ({}, "t")}
BATCH_SEED = 7
FIRST_GRAPH = {}                                                     # the first case's learned graph
TRAJ_SEED0 = 11


def put_dense_graph(g, key, a):
    """A dense [I, I] graph as its nonzero entries: `key.index` int32 [2, nnz] in row-major order and `key.values`."""
    a = a.detach().numpy()
    r, c = np.nonzero(a)
    g[key + ".index"], g[key + ".values"] = np.stack([r, c]).astype(np.int32), a[r, c].copy()


def grads(model):
    return {k: p.grad.numpy().copy() for k, p in model.named_parameters() if p.grad is not None}


def dump_model(g, prefix, overrides):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("LATTICE", dict(COMMON, **overrides))
    p = prefix
    if not prefix:
        inter = train_data.inter_matrix(form="coo")
        g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
        g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
        for k in ("embedding_size", "feat_embed_dim", "reg_weight", "learning_rate", "train_batch_size", "knn_k", "lambda_coeff"):
            g["cfg_" + k] = np.float64(config[k])
        na = model.norm_adj.coalesce()
        g["norm_adj_indices"], g["norm_adj_values"] = na.indices().numpy().astype(np.int32), na.values().numpy().copy()
    g[p + "cfg_cf_model"] = np.array(config["cf_model"])
    g[p + "cfg_n_layers"] = np.int64(config["n_layers"])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])
    if not prefix:                                                  # the same features in every case
        for name in ("image_original_adj", "text_original_adj"):
            put_dense_graph(g, name, getattr(model, name))

    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED); torch.manual_seed(BATCH_SEED)
    it = iter(train_data)
    batches = [next(it), next(it)]
    train_data.pr = 0
    seen = {}
    orig = model.forward

    def spy(adj, build_item_graph=False):
        out = orig(adj, build_item_graph=build_item_graph)
        seen["out"] = [o.detach().numpy().copy() for o in out]
        return out
    model.forward = spy
    model.train()
    model.pre_epoch_processing()
    for j, tag in enumerate(("build.", "plain.")):
        g[p + tag + "batch"] = batches[j].numpy().copy()
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(batches[j].clone())
        if tag == "build.":
            built = model.item_adj.detach().clone()
            if not prefix:
                FIRST_GRAPH["item_adj"] = built
                G.put(g, "build.u_g", seen["out"][0])
                G.put(g, "build.i_g", seen["out"][1])
            if not prefix or not torch.equal(built, FIRST_GRAPH["item_adj"]):
                put_dense_graph(g, p + "item_adj", built)
        loss.backward()
        g[p + tag + "loss"] = loss.detach().numpy().reshape(-1).copy()
        if tag == "build." or not prefix:
            for k, v in grads(model).items():
                G.put(g, p + tag + "grad." + k, v)
    del model.forward
    model.zero_grad(set_to_none=True)
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        g[p + "eval_users"], g[p + "eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        s = model.full_sort_predict(eb)
        G.put(g, p + "scores", s.numpy())
        # no optimizer step since the graph-building batch: evaluation leaves the same graph behind, bit for bit
        assert torch.equal(model.item_adj, built)
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10                                # trainer.py:304-309
        g[p + "topk50"] = torch.topk(m, 50, dim=-1)[1].numpy().astype(np.int16)
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g[p + "metric_names"] = np.array(list(res.keys()))
    g[p + "metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g[p + "test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)
    print(f"LATTICE{' ' + prefix if prefix else ''}: loss {float(g[p + 'build.loss'][0]):.6f} / {float(g[p + 'plain.loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("LATTICE", dict(COMMON))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())
        l = orig(interaction)
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    for ep in range(epochs):
        random.seed(TRAJ_SEED0 + ep); np.random.seed(TRAJ_SEED0 + ep); torch.manual_seed(TRAJ_SEED0 + ep)
        n0 = len(rec["batches"])
        model.pre_epoch_processing()                                 # as Trainer.fit does before each epoch
        trainer._train_epoch(train_data, ep)
        trainer.lr_scheduler.step()
        batch_epoch.append(len(rec["batches"]) - n0)
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    g = {"batch_sizes": np.array([b.shape[1] for b in rec["batches"]]), "batches": np.concatenate(rec["batches"], axis=1),
         "batches_per_epoch": np.array(batch_epoch), "losses": np.array(rec["losses"], dtype=np.float64),
         "valid": np.array(rec["valid"], dtype=np.float64), "test": np.array(rec["test"], dtype=np.float64),
         "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"]))}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    for k, v in model.state_dict().items():
        g["final." + k] = v.numpy().copy()
    np.savez_compressed(out, **g)
    print(f"trajectory LATTICE: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    g = {}
    u, i, e, dim, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.named("tiny")
    v, t = synth.make_features(i, f, seed=1)
    for prefix, (overrides, mods) in CASES.items():
        data_root = ref_loader.run_dir(os.path.join(tmp, "model_" + (prefix.rstrip(".") or "default")))
        synth.write_dataset(data_root, make_golden.DATASET, graph, v if "v" in mods else None, t if "t" in mods else None)
        dump_model(g, prefix, overrides)
        if not prefix:
            data_root = ref_loader.run_dir(os.path.join(tmp, "traj"))
            synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
            dump_trajectory(os.path.join(HERE, "traj_lattice_tiny.npz"))
    out = os.path.join(HERE, "lattice_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
