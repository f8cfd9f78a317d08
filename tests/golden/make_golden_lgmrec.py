"""Generate LGMRec's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF (src/models/lgmrec.py):

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_lgmrec.py

Same harness, dataset (`tiny`) and fields as make_golden.py's `dump_model` (which this file builds on and leaves unchanged),
plus `num_inters`, `adj` and every random draw.  LGMRec draws in every forward: four `F.gumbel_softmax` calls
(lgmrec.py:120-126, evaluation included) and, in training mode, four `nn.Dropout` masks (`:139-140`).  Both functions are
wrapped by restatements that consume torch's CPU generator exactly as torch does (`-empty_like().exponential_().log()`;
`empty_like().bernoulli_(1 - p).div_(1 - p)`) and record the Gumbel noise / the scaled mask; the generator asserts that the
wrapped run is bit-identical to an unwrapped run with the same seed.  The model files keep each phase's seed and, per
draw, its kind, shape and SHA-256 (`lgmrec_golden.py`); this generator asserts that a fresh CPU generator with that seed gives
exactly the draws the reference made, so the tests regenerate them (and check the digests) and replay them in order.  The
trajectory file keeps its draws themselves (H = 4: small).  The clothing file leaves out the fields bit-identical to the
default file's and names it (`lgmrec_golden.load` reads both).

Files: lgmrec_tiny.npz (the YAML's default, baby: H = 4, one hypergraph layer), lgmrec_clothing_tiny.npz (the YAML's
clothing comment: H = 64, two layers, keep rate 0.2, alpha 0.2), traj_lgmrec_tiny.npz (two epochs of the reference's
Trainer: batches, every draw in order, losses, per-epoch metrics).
"""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import lgmrec_golden  # noqa: E402
import make_golden  # noqa: E402
import ref_loader  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512}
SETTINGS = {"lgmrec_tiny.npz": {},
            "lgmrec_clothing_tiny.npz": {"n_hyper_layer": [2], "hyper_num": [64], "keep_rate": [0.2], "alpha": [0.2]}}
TRAJ = "traj_lgmrec_tiny.npz"
# torch seeds set before each recorded phase (the host test sets the same ones and must draw the same numbers)
SEEDS = {"fwd": 11, "loss": 4321, "scores": 12, "valid": 13, "test": 14}

_gumbel, _dropout = F.gumbel_softmax, F.dropout


class Recorder:
    """Restatements of `F.gumbel_softmax` (hard=False) and `F.dropout` that record their draws (torch 2.x CPU code path)."""

    def __init__(self):
        self.draws, self.specs = [], []

    def take(self, g, prefix, seed):
        """Store the phase drawn since the last call under `prefix`, after checking that it regenerates from `seed`."""
        g.update(lgmrec_golden.pack(prefix, seed, self.specs, self.draws))
        again = lgmrec_golden.regenerate(g, prefix)
        assert all(np.array_equal(a, b) for a, b in zip(again, self.draws)), prefix
        self.draws, self.specs = [], []

    def gumbel_softmax(self, logits, tau=1.0, hard=False, eps=1e-10, dim=-1):
        assert not hard
        gumbels = -torch.empty_like(logits, memory_format=torch.legacy_contiguous_format).exponential_().log()
        self.draws.append(gumbels.numpy().copy())
        self.specs.append(("gumbel", tuple(logits.shape), 0.0))
        return ((logits + gumbels) / tau).softmax(dim)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        assert not inplace
        if not training or p == 0 or input.numel() == 0:
            return input
        noise = torch.empty_like(input).bernoulli_(1 - p)
        noise.div_(1 - p)
        self.draws.append(noise.numpy().copy())
        self.specs.append(("dropout", tuple(input.shape), float(p)))
        return input * noise

    def __enter__(self):
        F.gumbel_softmax, F.dropout = self.gumbel_softmax, self.dropout
        return self

    def __exit__(self, *exc):
        F.gumbel_softmax, F.dropout = _gumbel, _dropout


def _put_draws(g, prefix, draws):
    g[prefix + "n_draws"] = np.int64(len(draws))
    for k, a in enumerate(draws):
        g["%sdraw%d" % (prefix, k)] = a


def dump_lgmrec(overrides, out, base=None):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("LGMRec", dict(COMMON, **overrides))
    g = {}
    inter = train_data.inter_matrix(form="coo")
    g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
    g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
    for k in ("embedding_size", "feat_embed_dim", "n_ui_layers", "n_mm_layers", "n_hyper_layer", "hyper_num", "keep_rate", "alpha",
              "cl_weight", "reg_weight", "train_batch_size"):
        g["cfg_" + k] = np.float64(config[k])
    g["norm_adj_idx"], g["norm_adj_val"] = make_golden.coo_parts(model.norm_adj)
    g["adj_idx"], g["adj_val"] = make_golden.coo_parts(model.adj)
    g["num_inters"] = model.num_inters.numpy().copy()
    for k, v in model.state_dict().items():
        g["param0." + k] = v.detach().numpy().copy()
    g["param_order"] = np.array([k for k, _ in model.named_parameters()])
    import random
    random.seed(7); np.random.seed(7)
    batch = next(iter(train_data))
    train_data.pr = 0
    g["batch"] = batch.numpy().copy()

    def eval_forward():
        model.eval()
        torch.manual_seed(SEEDS["fwd"])
        with torch.no_grad():
            return model.forward()

    def train_loss():
        model.train()
        torch.manual_seed(SEEDS["loss"])
        model.zero_grad()
        loss = model.calculate_loss(batch)
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        model.zero_grad()
        return loss.detach(), grads

    with Recorder() as rec:
        u, i, hyp = eval_forward()
        rec.take(g, "fwd_", SEEDS["fwd"])
        loss, grads = train_loss()
        rec.take(g, "loss_", SEEDS["loss"])
    # the restatements consume the generator exactly as torch's own functions: bit-identical results
    u2, i2, _ = eval_forward()
    loss2, grads2 = train_loss()
    assert torch.equal(u, u2) and torch.equal(i, i2) and torch.equal(loss, loss2)
    assert all(torch.equal(grads[k], grads2[k]) for k in grads)
    g["fwd_u"], g["fwd_i"] = u.numpy().copy(), i.numpy().copy()
    for name, h in zip(("uv", "iv", "ut", "it"), hyp):
        g["fwd_hyper_" + name] = h.numpy().copy()
    g["loss"] = loss.numpy().reshape(-1).copy()
    for k, v in grads.items():
        g["grad." + k] = v.numpy().copy()

    with Recorder() as rec:
        model.eval()
        torch.manual_seed(SEEDS["scores"])
        with torch.no_grad():
            eb = next(iter(valid_data))
            valid_data.pr = 0; valid_data.inter_pr = 0
            scores = model.full_sort_predict(eb)
        rec.take(g, "scores_", SEEDS["scores"])
        g["eval_users"], g["eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        g["scores"] = scores.numpy().copy()
        scores[eb[1][0], eb[1][1]] = -1e10
        tv, ti = torch.topk(scores, max(config["topk"]), dim=-1)
        g["topk_idx"], g["topk_val"] = ti.numpy().copy(), tv.numpy().copy()
        trainer = Trainer(config, model)
        torch.manual_seed(SEEDS["valid"])
        res = trainer.evaluate(valid_data)
        rec.take(g, "valid_", SEEDS["valid"])
        torch.manual_seed(SEEDS["test"])
        test_res = trainer.evaluate(test_data, is_test=True)
        rec.take(g, "test_", SEEDS["test"])
    g["metric_names"] = np.array(list(res.keys()))
    g["metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g["test_metric_values"] = np.array([test_res[k] for k in res], dtype=np.float64)
    if base is not None:
        g = lgmrec_golden.split_shared(g, dict(np.load(os.path.join(HERE, base), allow_pickle=True)), base)
    np.savez_compressed(out, **g)
    print(f"LGMRec {overrides}: wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB), loss {float(g['loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    """Two epochs of the reference's Trainer on its own LGMRec: every batch, every draw in order, every batch loss, metrics."""
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("LGMRec", dict(COMMON))
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
    torch.manual_seed(SEEDS["loss"])
    with Recorder() as r:
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
         "learning_rate": np.float64(config["learning_rate"])}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    _put_draws(g, "", r.draws)
    np.savez_compressed(out, **g)
    print(f"trajectory LGMRec: {len(rec['losses'])} batches, {len(r.draws)} draws, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)            # the CPU backward of torch.sparse.mm is only run-to-run reproducible on one thread
    ref_loader.install()
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    data_root = ref_loader.run_dir(tmp)
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    import logging
    logging.disable(logging.CRITICAL)
    first = None
    for name, over in SETTINGS.items():
        dump_lgmrec(over, os.path.join(HERE, name), base=first)
        first = first or name
    dump_trajectory(os.path.join(HERE, TRAJ))


if __name__ == "__main__":
    main()
