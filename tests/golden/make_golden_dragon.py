"""Generate DRAGON's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_dragon.py

The unmodified model class (`src/models/dragon.py`) runs under `ref_loader.install_pyg_shim()` (PyG's `MessagePassing`,
`degree`, `remove_self_loops`, restated from PyG's documented behaviour, as for DualGNN), with the harness, dataset and
fields of make_golden.py, `train_batch_size` 512, and the `user_graph_dict.npy` of `synth.write_user_graph_dict` (pinned
to the reference's preprocessing script by dualgnn_tiny.npz).  As for DualGNN, `result_embed` is unregistered after
construction and kept as a plain tensor: the reference registers it (`nn.Parameter(...).to(device)`, `dragon.py:155-156`)
only where `.to` returns its argument, on the CPU; on the GPU `.to` returns a plain tensor.  Each model is built in a
fresh data directory, so the constructor builds `mm_adj` instead of loading a `mm_adj_{k}.pt` left by another run.

Recorded (dragon_tiny.npz), each tensor as its SHA-256 and, where a tolerance applies, whole or as a fixed random sketch
(golden_io.put): the initial state as one SHA-256 per `state_dict` entry and of the float64 `result_embed`, the
parameter order, four `np.random` and four `torch` draws taken right after construction (`rng_after_*`: the
construction's RNG consumption), the coalesced `mm_adj` (indices and values), the seeded `pre_epoch_processing` sample;
on one batch in training mode `user_rep` before the user graph, `result_embed`, the mutated batch, the loss and every
gradient; the float64 scores before any forward (digest and the first SCORE_ROWS users' rows) and the scores after it,
the trainer's top-50 of those and the validation and test metrics.  Three models: both modalities (no prefix), text only
(`text.`) and `aggr_mode` 'mean' (`mean.`).
traj_dragon_tiny.npz: two epochs of the reference's Trainer (both modalities, 'add'), with `np.random` seeded before each
epoch's `pre_epoch_processing`."""
import os
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
# prefix -> (config overrides, text only)
CASES = {"": ({}, False), "text.": ({}, True), "mean.": ({"aggr_mode": "mean"}, False)}


def build(overrides=None):
    config, train_data, valid_data, test_data, model = make_golden.build("DRAGON", dict(COMMON, **(overrides or {})))
    r = model._parameters.pop("result_embed")                      # what `.to('cuda')` does (module docstring)
    model.result_embed = r.detach().clone()
    return config, train_data, valid_data, test_data, model


def rng_draws():
    """Four `np.random` and four `torch` draws, the generators' states restored after."""
    np_state, t_state = np.random.get_state(), torch.get_rng_state()
    a, b = np.random.randint(0, 2 ** 31, 4).astype(np.int64), torch.randint(0, 2 ** 31, (4,)).numpy()
    np.random.set_state(np_state)
    torch.set_rng_state(t_state)
    return a, b


def dump_model(g, prefix, overrides):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = build(overrides)
    p = prefix
    g[p + "rng_after_np"], g[p + "rng_after_torch"] = rng_draws()
    if not prefix:
        inter = train_data.inter_matrix(form="coo")
        g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
        g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
        for k in ("embedding_size", "reg_weight", "learning_rate", "train_batch_size", "knn_k", "mm_image_weight", "n_mm_layers"):
            g["cfg_" + k] = np.float64(config[k])
    g[p + "cfg_aggr_mode"] = np.array(config["aggr_mode"])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    assert model.result_embed.dtype == torch.float64
    g[p + "result_embed0_sha256"] = np.array(G.sha256_tagged(model.result_embed.numpy()))
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])
    mm = model.mm_adj.coalesce()
    g[p + "mm_adj_indices"] = mm.indices().numpy().copy()
    g[p + "mm_adj_values"] = mm.values().numpy().copy()
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
    print(f"DRAGON{' ' + prefix if prefix else ''}: loss {float(g[p + 'loss'][0]):.6f}")


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
    print(f"trajectory DRAGON: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    ref_loader.install_pyg_shim()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    g = {}
    u, i, e, dim, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.named("tiny")
    v, t = synth.make_features(i, f, seed=1)
    for prefix, (overrides, text_only) in CASES.items():
        data_root = ref_loader.run_dir(os.path.join(tmp, "model_" + (prefix.rstrip(".") or "both")))
        synth.write_dataset(data_root, make_golden.DATASET, graph, None if text_only else v, t)
        synth.write_user_graph_dict(data_root, make_golden.DATASET, graph)
        dump_model(g, prefix, overrides)
        if not prefix:
            dump_trajectory(os.path.join(HERE, "traj_dragon_tiny.npz"))
    out = os.path.join(HERE, "dragon_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
