"""Generate SELFCFED_LGN's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF (src/models/selfcfed_lgn.py,
src/common/encoders.py):

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_selfcf.py

Same harness and dataset (`tiny`) as make_golden_mvgae.py, `train_batch_size` 512.  Recorded:
- the initial state as one SHA-256 per `state_dict` entry (golden_io.init_digests);
- `sparse_norm_adj._indices()` and `_values()`: the stored entry order the encoder's dropout draws are applied in;
- on one batch, in training mode and seeded (numpy and torch seed SEEDS["loss"]): the forward's `u_online`, `i_online`, the
  loss and every gradient, with the SHA-256 of each draw (selfcf_golden.Replay) and the rate;
- the same phase for the model built with `n_layers` = 2 (the config's second value; fields `l2_*`): two dropped layers
  forward and the backward chain through both;
- `full_sort_predict` on the first validation batch and the Trainer's validation and test metrics;
- two epochs of the reference's Trainer with numpy and torch seeded TRAJ_SEED0 + b before batch b's `calculate_loss`: the
  batches, losses, draw digests and per-epoch metrics.
The generator asserts that a run under `Replay` is bit-identical to an unwrapped run with the same seeds (the restated
`F.dropout` consumes the CPU generator as torch's does).

Files: selfcfed_lgn_tiny.npz, traj_selfcfed_lgn_tiny.npz.
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
import selfcf_golden  # noqa: E402
from mmrec_b200.utils import synth  # noqa: E402

COMMON = {"eval_batch_size": 128, "train_batch_size": 512}
SEEDS = {"loss": 4321}
TRAJ_SEED0 = 6000


def _npz(g):
    """`g`'s init digests as an in-memory npz (for `golden_io.same_init`)."""
    import io
    buf = io.BytesIO()
    np.savez(buf, **{k: v for k, v in g.items() if k.startswith("init_sha256.")})
    buf.seek(0)
    return buf


def spy_rate(model, store):
    """Record the rate of every `sparse_dropout` call (the encoder passes `np.random.random() * drop_ratio`)."""
    enc = model.online_encoder
    orig = enc.sparse_dropout

    def sd(x, rate, noise_shape):
        store.append(float(rate))
        return orig(x, rate, noise_shape)
    enc.sparse_dropout = sd


def loss_phase(model, batch, prefix, g):
    """One seeded `calculate_loss` + backward, under `Replay` and again unwrapped (asserted bit-identical); its fields under
    `prefix`."""
    def train_loss(replay):
        model.train()
        model.zero_grad()
        rates, fwd = [], []
        spy_rate(model, rates)
        orig_fwd = model.forward

        def f(inputs):
            o = orig_fwd(inputs)
            fwd.append((o[0].detach().clone(), o[2].detach().clone()))
            return o
        model.forward = f
        if replay is None:
            np.random.seed(SEEDS["loss"]); torch.manual_seed(SEEDS["loss"])
            loss = model.calculate_loss(batch)
        else:
            with replay:
                loss = model.calculate_loss(batch)
        del model.forward
        del model.online_encoder.sparse_dropout
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        model.zero_grad()
        return loss.detach(), grads, rates, fwd

    rep = selfcf_golden.Replay(SEEDS["loss"])
    loss, grads, rates, fwd = train_loss(rep)
    loss2, grads2, rates2, fwd2 = train_loss(None)
    assert torch.equal(loss, loss2) and grads.keys() == grads2.keys() and all(torch.equal(grads[k], grads2[k]) for k in grads)
    assert rates == rates2 and len(rates) == 1 and len(rep.digests) == 3
    g[prefix + "loss_seed"] = np.int64(SEEDS["loss"])
    g[prefix + "loss_rate"] = np.float64(rates[0])
    g[prefix + "loss_draw_sha256"] = np.array(rep.digests)
    g[prefix + "fwd_u_online"], g[prefix + "fwd_i_online"] = fwd[0][0].numpy().copy(), fwd[0][1].numpy().copy()
    g[prefix + "loss"] = loss.numpy().reshape(-1).copy()
    for k, v in grads.items():
        g[prefix + "grad." + k] = v.numpy().copy()


def dump_selfcf(out):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("SELFCFED_LGN", dict(COMMON))
    g = {}
    inter = train_data.inter_matrix(form="coo")
    g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
    g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
    for k in ("embedding_size", "n_layers", "dropout", "reg_weight", "train_batch_size", "learning_rate"):
        g["cfg_" + k] = np.float64(config[k])
    for k, v in G.init_digests(model).items():
        g["init_sha256." + k] = np.array(v)
    g["param_order"] = np.array([k for k, _ in model.named_parameters()])
    adj = model.online_encoder.sparse_norm_adj
    g["adj_indices"] = adj._indices().numpy().copy()
    g["adj_values"] = adj._values().numpy().copy()
    import random
    random.seed(7); np.random.seed(7)
    batch = next(iter(train_data))
    train_data.pr = 0
    g["batch"] = batch.numpy().copy()
    loss_phase(model, batch, "", g)
    _, _, _, _, model2 = make_golden.build("SELFCFED_LGN", dict(COMMON, n_layers=2))
    assert model2.online_encoder.n_layers == 2 and not G.same_init(model2, np.load(_npz(g), allow_pickle=True))
    g["l2_cfg_n_layers"] = np.float64(2)
    loss_phase(model2, batch, "l2_", g)

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
    print(f"SELFCFED_LGN: wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB), loss {float(g['loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    """Two epochs of the reference's Trainer on its own SELFCFED_LGN: every batch, its draw digests and rate, every batch
    loss, per-epoch metrics."""
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("SELFCFED_LGN", dict(COMMON))
    config["epochs"] = epochs
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": [], "digests": [], "rates": []}
    orig = model.calculate_loss
    spy_rate(model, rec["rates"])

    def spy(interaction):
        b = len(rec["batches"])
        rec["batches"].append(interaction.numpy().copy())
        rep = selfcf_golden.Replay(TRAJ_SEED0 + b)
        with rep:
            l = orig(interaction)
        assert len(rep.digests) == 3
        rec["digests"].append(rep.digests)
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
         "learning_rate": np.float64(config["learning_rate"]), "n_steps": np.int64(len(rec["losses"])),
         "seed0": np.int64(TRAJ_SEED0), "draw_sha256": np.array(rec["digests"]), "rates": np.array(rec["rates"], dtype=np.float64)}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    np.savez_compressed(out, **g)
    print(f"trajectory SELFCFED_LGN: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    data_root = ref_loader.run_dir(tmp)
    u, i, e, d, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    import logging
    logging.disable(logging.CRITICAL)
    dump_selfcf(os.path.join(HERE, "selfcfed_lgn_tiny.npz"))
    dump_trajectory(os.path.join(HERE, "traj_selfcfed_lgn_tiny.npz"))


if __name__ == "__main__":
    main()
