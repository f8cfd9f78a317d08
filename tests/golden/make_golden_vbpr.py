"""Generate VBPR's and BPR's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_vbpr.py

The unmodified model classes (`src/models/vbpr.py`, `src/models/bpr.py`) run under the harness, dataset and fields of
make_golden.py (`tiny`, `train_batch_size` 512), with no shim.  vbpr_tiny.npz holds three VBPR cases under the prefixes of
`CASES` (both modalities, text only, image only), bpr_tiny.npz one BPR case under "bpr.".  Per case, each tensor is kept as
its SHA-256 and whole or as a fixed random sketch (golden_io.put):
- the SHA-256 of every initial `state_dict` entry, the parameter order and the torch RNG state after construction;
- one training batch, its [1]-shaped loss and every gradient;
- `full_sort_predict` of the first validation batch, the trainer's top-50 of it (int16), and the validation and test
  metrics.
traj_vbpr_tiny.npz / traj_bpr_tiny.npz: two epochs of the reference's Trainer (VBPR with both modalities), seeded
TRAJ_SEED0 + epoch before each epoch, with every batch, every loss, the per-epoch metrics and the final state; and whether
the torch RNG state was the same after every `calculate_loss` as before it (`F.dropout(·, 0.0)` draws nothing)."""
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
# prefix -> (model, modalities written to the dataset)
CASES = {"vt.": ("VBPR", "vt"), "t.": ("VBPR", "t"), "v.": ("VBPR", "v"), "bpr.": ("BPR", "")}
TRAJ = {"VBPR": "vt", "BPR": ""}
BATCH_SEED = 7
TRAJ_SEED0 = 21


def dump_model(g, prefix):
    from common.trainer import Trainer
    name, _ = CASES[prefix]
    config, train_data, valid_data, test_data, model = make_golden.build(name, dict(COMMON))
    p = prefix
    G.put_sha(g, p + "rng_after_init", torch.get_rng_state().numpy())
    g[p + "cfg"] = np.array([str(config["embedding_size"]), str(config["reg_weight"])])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])

    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED); torch.manual_seed(BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    g[p + "batch"] = batch.numpy().copy()
    model.train()
    model.zero_grad(set_to_none=True)
    loss = model.calculate_loss(batch.clone())
    loss.backward()
    g[p + "loss"] = loss.detach().numpy().reshape(-1).copy()
    g[p + "loss_shape"] = np.array(loss.shape, dtype=np.int64)
    for k, prm in model.named_parameters():
        if prm.grad is not None:
            G.put(g, p + "grad." + k, prm.grad.numpy())
    model.zero_grad(set_to_none=True)
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        g[p + "eval_users"], g[p + "eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        s = model.full_sort_predict(eb)
        G.put(g, p + "scores", s.numpy())
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10                                    # trainer.py:304-309
        g[p + "topk50"] = torch.topk(m, 50, dim=-1)[1].numpy().astype(np.int16)
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g[p + "metric_names"] = np.array(list(res.keys()))
    g[p + "metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g[p + "test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)
    print(f"{name} {prefix}: loss {float(g[p + 'loss'][0]):.6f}")


def dump_trajectory(name, out, epochs=2):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build(name, dict(COMMON))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": [], "rng_kept": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())
        st = torch.get_rng_state()
        l = orig(interaction)
        rec["rng_kept"].append(bool(torch.equal(st, torch.get_rng_state())))
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    for ep in range(epochs):
        random.seed(TRAJ_SEED0 + ep); np.random.seed(TRAJ_SEED0 + ep); torch.manual_seed(TRAJ_SEED0 + ep)
        n0 = len(rec["batches"])
        model.pre_epoch_processing()
        trainer._train_epoch(train_data, ep)
        trainer.lr_scheduler.step()
        batch_epoch.append(len(rec["batches"]) - n0)
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    g = {"batch_sizes": np.array([b.shape[1] for b in rec["batches"]]), "batches": np.concatenate(rec["batches"], axis=1),
         "batches_per_epoch": np.array(batch_epoch), "losses": np.array(rec["losses"], dtype=np.float64),
         "valid": np.array(rec["valid"], dtype=np.float64), "test": np.array(rec["test"], dtype=np.float64),
         "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"])),
         "rng_kept": np.array(rec["rng_kept"])}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    for k, v in model.state_dict().items():
        G.put(g, "final." + k, v.numpy())
    np.savez_compressed(out, **g)
    print(f"trajectory {name}: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    u, i, e, dim, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.named(make_golden.DATASET)
    v, t = synth.make_features(i, f, seed=1)
    files = {"VBPR": {}, "BPR": {}}
    for prefix, (name, mods) in CASES.items():
        data_root = ref_loader.run_dir(os.path.join(tmp, "model_" + prefix.rstrip(".")))
        synth.write_dataset(data_root, make_golden.DATASET, graph, v if "v" in mods else None, t if "t" in mods else None)
        dump_model(files[name], prefix)
    for name, mods in TRAJ.items():
        data_root = ref_loader.run_dir(os.path.join(tmp, "traj_" + name))
        synth.write_dataset(data_root, make_golden.DATASET, graph, v if "v" in mods else None, t if "t" in mods else None)
        dump_trajectory(name, os.path.join(HERE, f"traj_{name.lower()}_tiny.npz"))
    for name, g in files.items():
        out = os.path.join(HERE, f"{name.lower()}_tiny.npz")
        np.savez_compressed(out, **g)
        print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
