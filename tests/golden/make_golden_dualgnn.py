"""Generate DualGNN's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_dualgnn.py

1. The unmodified preprocessing script `preprocessing/dualgnn-gen-u-u-matrix.py` runs as a program on `tiny` and on the
   small tie-heavy graph `dualgnn_golden.GRAPHS['ties']`.  It `chdir`s to `../src` and reads `configs/overall.yaml`,
   `configs/dataset/<name>.yaml` and `../data/<name>/`, so each run gets a temporary tree laid out that way, with a dataset
   yaml naming the synthetic file's columns.  Its `user_graph_dict.npy` is kept as the digests of its flat arrays
   (dualgnn_golden.flatten).
2. The unmodified model class (`src/models/dualgnn.py`) runs under `ref_loader.install_pyg_shim()` (PyG's
   `MessagePassing`, `degree`, `remove_self_loops`, restated from PyG's documented behaviour; as for MMGCN and MVGAE, PyG
   itself is unpinned and the shim's formula is what is pinned), with the same harness, dataset and fields as
   make_golden.py, `train_batch_size` 512, and the script's `user_graph_dict.npy` of `tiny`.  One further shim: after
   construction `result_embed` is unregistered and kept as a plain tensor.  The reference registers it as a parameter
   (`nn.Parameter(...).to(device)`, `dualgnn.py:129`) only where `.to` returns its argument, on the CPU; on the GPU `.to`
   returns a plain tensor.  Without the shim its own `forward` raises `TypeError` on the CPU (`:174` assigns a tensor to
   a parameter's name).

Recorded (dualgnn_tiny.npz), each tensor as its SHA-256 and, where a tolerance applies, whole or as a fixed random
sketch (golden_io.put): both user-graph dicts (digests of their flat arrays); the initial state as one SHA-256 per
`state_dict` entry and of the float64 `result_embed`, and the parameter order; the seeded `pre_epoch_processing` sample
(index and weights); on one batch in training mode `v_rep` / `t_rep` after the in-place add, `user_rep` before the user
graph, `result_embed` (whole), the mutated batch, the loss and every gradient; the float64 scores before any forward
(digest, and the first SCORE_ROWS users' rows) and the scores after it (whole), the trainer's top-50 of those and the
validation and test metrics; the same for the text-only model (`text.` prefix; its `result_embed` and scores sketched).
traj_dualgnn_tiny.npz: two epochs of the reference's Trainer, with `np.random` seeded before each epoch's
`pre_epoch_processing`.

DualGNN's training forward draws nothing at random; `pre_epoch_processing` draws its padding from `np.random`."""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import dualgnn_golden as D  # noqa: E402
import golden_io as G  # noqa: E402
import make_golden  # noqa: E402
import ref_loader  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512, "user_graph_dict_file": "user_graph_dict.npy"}
SCORE_ROWS = 16


def graph_of(name):
    return synth.named(name) if D.GRAPHS[name] is None else synth.make_graph(*D.GRAPHS[name])


def run_script(tmp, name, graph):
    """The preprocessing script, unmodified, as a program; returns the path of the file it wrote."""
    root = os.path.join(tmp, "script_" + name)
    os.makedirs(os.path.join(root, "preprocessing"))
    os.makedirs(os.path.join(root, "src", "configs", "dataset"))
    os.symlink(os.path.join(ref_loader.REF_SRC, "configs", "overall.yaml"), os.path.join(root, "src", "configs", "overall.yaml"))
    with open(os.path.join(root, "src", "configs", "dataset", name + ".yaml"), "w") as f:
        f.write(f"USER_ID_FIELD: userID\nITEM_ID_FIELD: itemID\ninter_file_name: '{name}.inter'\n"
                "user_graph_dict_file: 'user_graph_dict.npy'\n")
    synth.write_dataset(os.path.join(root, "data"), name, graph)
    script = os.path.join(os.path.dirname(os.path.abspath(ref_loader.REF_SRC)), "preprocessing", "dualgnn-gen-u-u-matrix.py")
    subprocess.run([sys.executable, script, "-d", name], cwd=os.path.join(root, "preprocessing"), check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return os.path.join(root, "data", name, "user_graph_dict.npy")


def build(overrides=None):
    config, train_data, valid_data, test_data, model = make_golden.build("DualGNN", dict(COMMON, **(overrides or {})))
    r = model._parameters.pop("result_embed")                      # what `.to('cuda')` does (module docstring)
    model.result_embed = r.detach().clone()
    return config, train_data, valid_data, test_data, model


def dump_model(g, prefix):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = build()
    p = prefix
    if not prefix:
        inter = train_data.inter_matrix(form="coo")
        g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
        g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
        for k in ("embedding_size", "reg_weight", "learning_rate", "train_batch_size"):
            g["cfg_" + k] = np.float64(config[k])
        g["cfg_aggr_mode"] = np.array(config["aggr_mode"])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    assert model.result_embed.dtype == torch.float64
    g[p + "result_embed0_sha256"] = np.array(G.sha256_tagged(model.result_embed.numpy()))
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])
    model.eval()
    with torch.no_grad():                                           # before any forward: the float64 initial table
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        g[p + "eval_users"], g[p + "eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        s0 = model.full_sort_predict(eb)
        assert s0.dtype == torch.float64
        G.put_sha(g, p + "scores0", s0.numpy())
        g[p + "scores0_rows"] = s0[:SCORE_ROWS].numpy().copy()
    np.random.seed(D.SAMPLE_SEED)
    model.pre_epoch_processing()
    G.put_sha(g, p + "sample_idx", np.array(model.epoch_user_graph, dtype=np.int64))
    G.put_sha(g, p + "sample_w", model.user_weight_matrix.numpy())
    import random
    random.seed(D.BATCH_SEED); np.random.seed(D.BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    g[p + "batch"] = batch.numpy().copy()
    seen = {}
    orig = model.user_graph.forward

    def spy(features, user_graph, user_matrix):
        seen["user_rep"] = features.detach().numpy().copy()
        return orig(features, user_graph, user_matrix)
    model.user_graph.forward = spy
    model.train()
    model.zero_grad()
    b = batch.clone()
    loss = model.calculate_loss(b)
    del model.user_graph.forward
    g[p + "batch_after"] = b.numpy().copy()
    G.put(g, p + "user_rep", seen["user_rep"])
    for name in ("v_rep", "t_rep"):
        if getattr(model, name) is not None:
            G.put(g, p + name, getattr(model, name).detach().squeeze(2).numpy())
    G.put(g, p + "result_embed", model.result_embed.detach().numpy(), whole=not prefix)
    loss.backward()
    g[p + "loss"] = loss.detach().numpy().reshape(-1).copy()
    for k, prm in model.named_parameters():
        if prm.grad is not None:
            G.put(g, p + "grad." + k, prm.grad.numpy())
    model.zero_grad()
    model.eval()
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        G.put(g, p + "scores", s.numpy(), whole=not prefix)
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10                                # trainer.py:304-309
        g[p + "topk50"] = torch.topk(m, 50, dim=-1)[1].numpy().copy()
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g[p + "metric_names"] = np.array(list(res.keys()))
    g[p + "metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g[p + "test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)
    print(f"DualGNN{' ' + prefix if prefix else ''}: loss {float(g[p + 'loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = build()
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())             # before forward's in-place offset
        l = orig(interaction)
        rec["losses"].append(float(l))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    for ep in range(epochs):
        np.random.seed(D.EPOCH_SEED0 + ep)
        model.pre_epoch_processing()
        n0 = len(rec["batches"])
        trainer._train_epoch(train_data, ep)
        trainer.lr_scheduler.step()
        batch_epoch.append(len(rec["batches"]) - n0)
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    g = {"batch_sizes": np.array([b.shape[1] for b in rec["batches"]]), "batches": np.concatenate(rec["batches"], axis=1),
         "batches_per_epoch": np.array(batch_epoch), "losses": np.array(rec["losses"], dtype=np.float64),
         "valid": np.array(rec["valid"], dtype=np.float64), "test": np.array(rec["test"], dtype=np.float64),
         "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"])),
         "epoch_seed0": np.int64(D.EPOCH_SEED0)}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    np.savez_compressed(out, **g)
    print(f"trajectory DualGNN: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    ref_loader.install_pyg_shim()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    g = {}
    files = {}
    for name in D.GRAPHS:
        files[name] = run_script(tmp, name, graph_of(name))
        d = np.load(files[name], allow_pickle=True).item()
        for part, a in zip(("ptr", "idx", "val"), D.flatten(d)):
            G.put_sha(g, "ugd_%s_%s" % (name, part), a)
    u, i, e, dim, f = synth.SHAPES[make_golden.DATASET]
    graph = graph_of("tiny")
    v, t = synth.make_features(i, f, seed=1)
    for prefix, feats in (("", (v, t)), ("text.", (None, t))):
        data_root = ref_loader.run_dir(os.path.join(tmp, "model_" + (prefix or "both")))
        synth.write_dataset(data_root, make_golden.DATASET, graph, *feats)
        shutil.copy(files["tiny"], os.path.join(data_root, make_golden.DATASET, "user_graph_dict.npy"))
        dump_model(g, prefix)
        if not prefix:
            dump_trajectory(os.path.join(HERE, "traj_dualgnn_tiny.npz"))
    out = os.path.join(HERE, "dualgnn_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
