"""Generate MMGCF's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_mmgcf.py

The unmodified model class (`src/models/mmgcf.py`) runs under the harness, dataset and fields of make_golden.py (`tiny`,
`train_batch_size` 512), with no shim.  For every case of `CASES` (all nine fusion_mode x weighting pairs with both
modalities, two pairs text-only; n_ui_layers 1 or 2) mmgcf_tiny.npz keeps, under the case's name as prefix, each tensor as
its SHA-256 and, where a tolerance applies, whole or as a fixed random sketch (golden_io.put):
- the initial state, one SHA-256 per `state_dict` entry, and the parameter order;
- once for all cases (they are the same): `norm_adj` and the masked adjacency (digests of the COO indices, values whole),
  `edge_values`, and the pruning draw (`torch.multinomial` with torch seeded PRUNE_SEED, recorded from a saved RNG state
  and then drawn again by `pre_epoch_processing` itself);
- `forward` on `norm_adj` and on the masked adjacency: the item rows, and the user rows on `norm_adj` in the USER_ROWS
  cases (one per n_ui_layers; they do not depend on the fusion);
- once for all cases: the recorded training batch and the first validation batch (users and mask);
- one batch's loss and every gradient;
- `full_sort_predict` on the first validation batch, the trainer's top-50 of it (int16), and the validation and test
  metrics.
traj_mmgcf_<case>_tiny.npz: two epochs of the reference's Trainer with pruning (dropout 0.2) for one element-wise and
one concat pair, torch seeded TRAJ_SEED0 + epoch before each epoch's `pre_epoch_processing`, every batch, every loss, each
epoch's pruning draw and the per-epoch metrics."""
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
PRUNE_SEED = 1234
BATCH_SEED = 7
TRAJ_SEED0 = 5000
# name -> (fusion_mode, weighting, n_ui_layers, text only)
CASES = {f"{f}_{w}": (f, w, 1 + k % 2, False)
         for k, (f, w) in enumerate((f, w) for f in ("mean", "sum", "concat") for w in ("equal", "alpha", "normalized"))}
CASES.update({"text_mean_alpha": ("mean", "alpha", 2, True), "text_concat_equal": ("concat", "equal", 1, True)})
USER_ROWS = ("mean_equal", "mean_alpha")                           # n_ui_layers 1 and 2
TRAJ = {"mean_normalized": ("mean", "normalized"), "concat_alpha": ("concat", "alpha")}
TRAJ_DROPOUT = 0.2


def overrides(fusion, weighting, layers, dropout=None):
    o = dict(COMMON, fusion_mode=[fusion], weighting=[weighting], n_ui_layers=[layers])
    if dropout is not None:
        o["dropout"] = [dropout]
    return o


def keep_draw(model):
    """The `torch.multinomial` draw the next `pre_epoch_processing` makes, without consuming it."""
    keep_len = int(model.edge_values.size(0) * (1.0 - model.dropout))
    st = torch.get_rng_state()
    k = torch.multinomial(model.edge_values, keep_len).numpy().copy()
    torch.set_rng_state(st)
    return k


def dump_case(g, name):
    from common.trainer import Trainer
    fusion, weighting, layers, _ = CASES[name]
    config, train_data, valid_data, test_data, model = make_golden.build("MMGCF", overrides(fusion, weighting, layers))
    p = name + "."
    g[p + "cfg"] = np.array([fusion, weighting, str(layers), str(config["dropout"]), str(config["reg_weight"])])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])
    torch.manual_seed(PRUNE_SEED)
    keep = keep_draw(model)
    model.pre_epoch_processing()
    if "norm_adj_val.sha256" not in g:                                 # the same graphs and draw in every case
        g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
        for tag, adj in (("norm_adj", model.norm_adj), ("masked_adj", model.masked_adj)):
            idx, val = make_golden.coo_parts(adj)
            G.put_sha(g, tag + "_idx", idx)
            G.put(g, tag + "_val", val, whole=True)
        G.put(g, "edge_values", model.edge_values.numpy(), whole=True)
        g["prune_keep_idx"] = keep
    assert np.array_equal(keep, g["prune_keep_idx"])
    import random
    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    g.setdefault("batch", batch.numpy().copy())
    assert np.array_equal(batch.numpy(), g["batch"])
    model.eval()
    with torch.no_grad():
        for tag, adj in (("fwd", model.norm_adj), ("fwd_masked", model.masked_adj)):
            u, i = model.forward(adj)
            if tag == "fwd" and name in USER_ROWS:                     # the user rows do not depend on the fusion
                G.put(g, p + tag + "_u", u.numpy())
            G.put(g, p + tag + "_i", i.numpy())
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(batch)
    loss.backward()
    g[p + "loss"] = loss.detach().numpy().reshape(-1).copy()
    for k, prm in model.named_parameters():
        if prm.grad is not None:
            G.put(g, p + "grad." + k, prm.grad.numpy())
    model.zero_grad()
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        g.setdefault("eval_users", eb[0].numpy().copy())
        g.setdefault("eval_mask", eb[1].numpy().copy())
        assert np.array_equal(eb[0].numpy(), g["eval_users"]) and np.array_equal(eb[1].numpy(), g["eval_mask"])
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
    print(f"MMGCF {name}: loss {float(g[p + 'loss'][0]):.6f}")


def dump_trajectory(name, out, epochs=2):
    from common.trainer import Trainer
    fusion, weighting = TRAJ[name]
    config, train_data, valid_data, test_data, model = make_golden.build("MMGCF", overrides(fusion, weighting, 2, TRAJ_DROPOUT))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": [], "keep": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())
        l = orig(interaction)
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    for ep in range(epochs):
        torch.manual_seed(TRAJ_SEED0 + ep)
        rec["keep"].append(keep_draw(model))
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
         "keep_idx": np.stack(rec["keep"]), "learning_rate": np.float64(config["learning_rate"]),
         "n_steps": np.int64(len(rec["losses"])), "seed0": np.int64(TRAJ_SEED0), "dropout": np.float64(TRAJ_DROPOUT),
         "cfg": np.array([fusion, weighting])}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    np.savez_compressed(out, **g)
    print(f"trajectory MMGCF {name}: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.named(make_golden.DATASET)
    v, t = synth.make_features(i, f, seed=1)
    g = {}
    for text_only in (False, True):
        data_root = ref_loader.run_dir(os.path.join(tmp, "text" if text_only else "both"))
        synth.write_dataset(data_root, make_golden.DATASET, graph, None if text_only else v, t)
        for name, case in CASES.items():
            if case[3] == text_only:
                dump_case(g, name)
        if not text_only:
            for name in TRAJ:
                dump_trajectory(name, os.path.join(HERE, f"traj_mmgcf_{name}_tiny.npz"))
    out = os.path.join(HERE, "mmgcf_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
