"""Generate SLMRec's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF (src/models/slmrec.py):

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_slmrec.py

Same harness and dataset (`tiny`) as make_golden_selfcf.py, `train_batch_size` 512, every grid key at its first value.
`slmrec.py` imports `torch_scatter.scatter` at module top; the shim gets a stub of it (never called under FAC).  FAC draws
nothing at random, so only the batching is seeded.  Recorded:
- the initial state as one SHA-256 per `state_dict` entry (golden_io.init_digests) and the parameter order;
- `norm_adj._indices()` and `_values()` (`adj_type: pre`);
- on one batch, in training mode: the three views `i_emb`, `v_emb`, `t_emb` of `compute()`, the loss and every gradient;
- `full_sort_predict` on the first validation batch (the tables of that last `calculate_loss`) and the Trainer's
  validation and test metrics;
- two epochs of the reference's Trainer: the batches, the losses and the per-epoch metrics.

Files: slmrec_tiny.npz, traj_slmrec_tiny.npz.
"""
import os
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
BATCH_SEED = 7


def dump_slmrec(out):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("SLMRec", dict(COMMON))
    g = {}
    inter = train_data.inter_matrix(form="coo")
    g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
    g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
    for k in ("recdim", "layer_num", "ssl_temp", "ssl_alpha", "temp", "learning_rate", "weight_decay", "train_batch_size"):
        g["cfg_" + k] = np.float64(config[k])
    g["cfg_adj_type"] = np.array(config["adj_type"])
    for k, v in G.init_digests(model).items():
        g["init_sha256." + k] = np.array(v)
    g["param_order"] = np.array([k for k, _ in model.named_parameters()])
    g["adj_indices"] = model.norm_adj._indices().numpy().copy()
    g["adj_values"] = model.norm_adj._values().numpy().copy()
    import random
    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    g["batch"] = batch.numpy().copy()
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(batch)
    for name in ("i_emb", "v_emb", "t_emb"):
        g["view_" + name] = getattr(model, name).detach().numpy().copy()
    g["all_users"] = model.all_users.detach().numpy().copy()
    g["all_items"] = model.all_items.detach().numpy().copy()
    loss.backward()
    g["loss"] = loss.detach().numpy().reshape(-1).copy()
    for k, p in model.named_parameters():
        if p.grad is not None:
            g["grad." + k] = p.grad.numpy().copy()
    model.zero_grad()

    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        scores = model.full_sort_predict(eb)
        g["eval_users"], g["eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        g["scores"] = scores.numpy().copy()
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g["metric_names"] = np.array(list(res.keys()))
    g["metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g["test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)
    np.savez_compressed(out, **g)
    print(f"SLMRec: wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB), loss {float(g['loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    """Two epochs of the reference's Trainer on its own SLMRec: every batch, every batch loss, per-epoch metrics."""
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("SLMRec", dict(COMMON))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())
        l = orig(interaction)
        rec["losses"].append(float(l))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    for ep in range(epochs):
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
         "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"]))}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    np.savez_compressed(out, **g)
    print(f"trajectory SLMRec: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    sys.modules["torch_scatter"].scatter = lambda *a, **k: None     # imported by slmrec.py:13, used only by a commented-out branch
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    data_root = ref_loader.run_dir(tmp)
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    import logging
    logging.disable(logging.CRITICAL)
    dump_slmrec(os.path.join(HERE, "slmrec_tiny.npz"))
    dump_trajectory(os.path.join(HERE, "traj_slmrec_tiny.npz"))


if __name__ == "__main__":
    main()
