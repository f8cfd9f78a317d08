"""Generate MVGAE's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF (src/models/mvgae.py):

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_mvgae.py

The reference's file imports torch_geometric; it runs unmodified under `ref_loader.install_pyg_shim()` (the PyG primitives
it uses -- `MessagePassing`, `remove_self_loops`, `add_self_loops`, `degree`, `inits.uniform` -- restated from PyG's
documented behaviour, as for MMGCN).  Same harness, dataset (`tiny`) and fields as make_golden.py's `dump_model`, with
`train_batch_size` 512, except where that would make the file large:
- the initial state (the `state_dict` and the plain tensors the reference keeps beside its parameters: `collaborative`,
  each GCN's `preference`, the initial `result_embed`) is kept as one SHA-256 per tensor (`golden_io.init_digests`: bit
  for bit, without 1.2 MiB of incompressible weights);
- the forward keeps its output `pd_mu`, the precision-weighted mean of the experts, which every tower's mu and logvar enter
  (in evaluation mode z is pd_mu; pd_logvar enters the recorded loss and gradients);
- the trainer's top-50 is left to the recorded metrics.
Plus the value and argmax of every `dot_product_decode_neg` call of the recorded loss, and every random draw.

Draws: a training forward draws three `F.dropout` masks per GCN (v, t, c) and four `torch.randn_like` tensors (z, z_v, z_t,
z_c).  Both functions are wrapped by restatements that consume torch's CPU generator exactly as torch does
(`empty_like().bernoulli_(1 - p).div_(1 - p)`; `empty_like().normal_()`) and record the draws; the generator asserts that
the wrapped run is bit-identical to an unwrapped run with the same seed, and that a fresh CPU generator with the phase's
seed regenerates every draw (mvgae_golden.py), so the files keep the seed and a SHA-256 per draw.  The trajectory (two
epochs of the reference's Trainer) seeds torch before each batch's `calculate_loss` (seed TRAJ_SEED0 + batch) and keeps one
such phase per batch: its draws are 3 MiB of incompressible noise at `tiny`.

Files: mvgae_tiny.npz, traj_mvgae_tiny.npz.
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

import golden_io as G  # noqa: E402
import lgmrec_golden  # noqa: E402
import make_golden  # noqa: E402
import mvgae_golden  # noqa: E402
import ref_loader  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512}
SEEDS = {"loss": 4321}
TRAJ_SEED0 = 5000

_dropout, _randn_like = F.dropout, torch.randn_like


class Recorder:
    """Restatements of `F.dropout` and `torch.randn_like` (torch 2.x CPU code path) that record their draws."""

    def __init__(self):
        self.draws, self.specs = [], []

    def take(self, g, prefix, seed):
        """Store the phase drawn since the last call under `prefix`, after checking that it regenerates from `seed`."""
        g.update(lgmrec_golden.pack(prefix, seed, self.specs, self.draws))
        again = mvgae_golden.regenerate(g, prefix)
        assert len(again) == len(self.draws) and all(np.array_equal(a, b) for a, b in zip(again, self.draws)), prefix
        self.draws, self.specs = [], []

    def dropout(self, input, p=0.5, training=True, inplace=False):
        assert not inplace
        if not training or p == 0 or input.numel() == 0:
            return input
        noise = torch.empty_like(input).bernoulli_(1 - p)
        noise.div_(1 - p)
        self.draws.append(noise.numpy().copy())
        self.specs.append(("dropout", tuple(input.shape), float(p)))
        return input * noise

    def randn_like(self, input, **kw):
        assert not kw
        x = torch.empty_like(input).normal_()
        self.draws.append(x.numpy().copy())
        self.specs.append(("randn", tuple(input.shape), 0.0))
        return x

    def __enter__(self):
        F.dropout, torch.randn_like = self.dropout, self.randn_like
        return self

    def __exit__(self, *exc):
        F.dropout, torch.randn_like = _dropout, _randn_like


def spy_decode(model, store):
    """Wrap `dot_product_decode_neg` to record, per call, the max over the batch's negatives and its first argmax, computed
    with the reference's own expression (mvgae.py:76-84)."""
    orig = model.dot_product_decode_neg

    def decode(z, user, neg_items, sigmoid=True):
        out = orig(z, user, neg_items, sigmoid)
        with torch.no_grad():
            neg_values = torch.sum(z[torch.unsqueeze(user, 1).repeat(1, neg_items.size(0))] * z[neg_items], -1)
            v, i = torch.max(neg_values, dim=-1)
        store.append((v.numpy().copy(), i.numpy().copy()))
        return out
    model.dot_product_decode_neg = decode
    return orig


def dump_mvgae(out):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("MVGAE", dict(COMMON))
    g = {}
    inter = train_data.inter_matrix(form="coo")
    g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
    g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
    for k in ("embedding_size", "n_layers", "beta", "train_batch_size", "learning_rate"):
        g["cfg_" + k] = np.float64(config[k])
    g["edge_index"] = model.edge_index.numpy().copy()
    for k, v in G.init_digests(model, mvgae_golden.plain(model)).items():
        g["init_sha256." + k] = np.array(v)
    g["param_order"] = np.array([k for k, _ in model.named_parameters()])
    import random
    random.seed(7); np.random.seed(7)
    batch = next(iter(train_data))
    train_data.pr = 0
    g["batch"] = batch.numpy().copy()

    def train_loss(decodes=None):
        model.train()
        torch.manual_seed(SEEDS["loss"])
        model.zero_grad()
        orig = spy_decode(model, decodes) if decodes is not None else None
        loss = model.calculate_loss(batch)
        if orig is not None:
            del model.dot_product_decode_neg                          # back to the class's method
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        model.zero_grad()
        return loss.detach(), grads

    with Recorder() as rec:
        model.eval()
        with torch.no_grad():
            fwd = model.forward()
        assert not rec.draws                                          # evaluation mode draws nothing
        decodes = []
        loss, grads = train_loss(decodes)
        rec.take(g, "loss_", SEEDS["loss"])
    loss2, grads2 = train_loss()
    assert torch.equal(loss, loss2) and grads.keys() == grads2.keys() and all(torch.equal(grads[k], grads2[k]) for k in grads)
    assert torch.equal(fwd[2], fwd[0])                                 # evaluation mode: z is pd_mu
    g["fwd_pd_mu"] = fwd[0].numpy().copy()
    g["loss"] = loss.numpy().reshape(-1).copy()
    for k, v in grads.items():
        g["grad." + k] = v.numpy().copy()
    assert len(decodes) == 4
    g["decode_val"] = np.stack([v for v, _ in decodes])
    g["decode_arg"] = np.stack([i for _, i in decodes])

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
    print(f"MVGAE: wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB), loss {float(g['loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    """Two epochs of the reference's Trainer on its own MVGAE: every batch, its seed and draw digests, every batch loss,
    per-epoch metrics."""
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("MVGAE", dict(COMMON))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": []}
    g = {}
    orig = model.calculate_loss
    r = Recorder()

    def spy(interaction):
        b = len(rec["batches"])
        rec["batches"].append(interaction.numpy().copy())
        torch.manual_seed(TRAJ_SEED0 + b)
        l = orig(interaction)
        r.take(g, "step%d_" % b, TRAJ_SEED0 + b)
        rec["losses"].append(float(l))
        return l
    model.calculate_loss = spy
    batch_epoch = []
    with r:
        for ep in range(epochs):
            model.pre_epoch_processing()
            n0 = len(rec["batches"])
            trainer._train_epoch(train_data, ep)
            trainer.lr_scheduler.step()
            batch_epoch.append(len(rec["batches"]) - n0)
            rec["valid"].append(list(trainer.evaluate(valid_data).values()))
            rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    g.update({"batch_sizes": np.array([b.shape[1] for b in rec["batches"]]), "batches": np.concatenate(rec["batches"], axis=1),
              "batches_per_epoch": np.array(batch_epoch), "losses": np.array(rec["losses"], dtype=np.float64),
              "valid": np.array(rec["valid"], dtype=np.float64), "test": np.array(rec["test"], dtype=np.float64),
              "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"]))})
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    np.savez_compressed(out, **g)
    print(f"trajectory MVGAE: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    ref_loader.install_pyg_shim()
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    data_root = ref_loader.run_dir(tmp)
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    import logging
    logging.disable(logging.CRITICAL)
    dump_mvgae(os.path.join(HERE, "mvgae_tiny.npz"))
    dump_trajectory(os.path.join(HERE, "traj_mvgae_tiny.npz"))


if __name__ == "__main__":
    main()
