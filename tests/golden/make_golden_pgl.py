"""Generate PGL's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_pgl.py

The unmodified `src/models/pgl.py` runs under the harness, dataset and fields of make_golden.py (`tiny`,
`train_batch_size` 512) in its shipped configuration (`mode: local`).  One stub: `pgl.py` imports `sparsesvd` at module top
(`:19`), a package the reference's requirements do not list; only the global mode calls it, so an empty module named
`sparsesvd` whose function raises is put in `sys.modules` before the import.

pgl_tiny.npz (each tensor kept as its SHA-256 and whole or as a fixed random sketch, golden_io.put):
- the SHA-256 of every initial `state_dict` entry, the parameter order and the torch RNG state after construction;
- the epoch's keep indices (`torch.multinomial(edge_values, int(nnz * 0.3))` after `torch.manual_seed(PRUNE_SEED)`);
- `forward` on the sub-graph and on `norm_adj`;
- one training batch and, after `torch.manual_seed(LOSS_SEED)`, the four dropout masks of its `calculate_loss` (captured
  by hooks on `model.dropoutf`: the draw is replayed from the generator state before the call and checked against the
  output, then packed as bits), and the 0-dim loss and every gradient at reg_weight 0 (`rw0.`) and 0.1 (`rw1.`);
- `full_sort_predict` of the first validation batch, the trainer's top-50 of it (int16), and the validation and test metrics.
traj_pgl_tiny.npz: two epochs of the reference's Trainer at dropout 0.0 and reg_weight 0.1, seeded TRAJ_SEED0 + epoch
before each epoch, with every batch, every loss, each epoch's keep indices, the per-epoch metrics and the final state."""
import os
import random
import sys
import tempfile
import types

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
REG_CASES = {"rw0.": 0.0, "rw1.": 0.1}
TRAJ_OVER = {"dropout": [0.0], "reg_weight": [0.1]}
BATCH_SEED = 7
PRUNE_SEED = 1234
LOSS_SEED = 4321
TRAJ_SEED0 = 21


def install_sparsesvd_stub():
    def sparsesvd(*_a, **_k):
        raise RuntimeError("sparsesvd stub: only PGL's global mode calls it")
    mod = types.ModuleType("sparsesvd")
    mod.sparsesvd = sparsesvd
    sys.modules.setdefault("sparsesvd", mod)


def keep_len(model):
    return int(model.edge_values.size(0) * 0.3)


def draw_keep(model):
    """The keep indices the next `pre_epoch_processing` draws (the generator state is restored after the draw)."""
    st = torch.get_rng_state()
    keep = torch.multinomial(model.edge_values, keep_len(model)).numpy().copy()
    torch.set_rng_state(st)
    return keep


class MaskSpy:
    """The bool masks of every `model.dropoutf` call, replayed from the generator state before the call (CPU dropout is
    `noise.bernoulli_(1 - p)`, `noise / (1 - p)`, `input * noise`) and checked against the call's output."""

    def __init__(self, module):
        self.masks, self.state = [], None
        self.p = module.p
        module.register_forward_pre_hook(self.pre)
        module.register_forward_hook(self.post)

    def pre(self, mod, inp):
        self.state = torch.get_rng_state()

    def post(self, mod, inp, out):
        if not mod.training or self.p == 0:
            return
        cur = torch.get_rng_state()
        torch.set_rng_state(self.state)
        noise = torch.empty_like(inp[0]).bernoulli_(1 - self.p)
        torch.set_rng_state(cur)
        assert torch.equal(inp[0] * noise.div(1 - self.p), out), "dropout replay differs from the call"
        self.masks.append((noise != 0).numpy().copy())


def dump_model(g):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("PGL", dict(COMMON))
    G.put_sha(g, "rng_after_init", torch.get_rng_state().numpy())
    g["cfg"] = np.array([str(config[k]) for k in ("embedding_size", "feat_embed_dim", "dropout", "reg_weight", "mode",
                                                   "n_mm_layers", "n_ui_layers", "knn_k", "mm_image_weight")])
    for k, v in G.init_digests(model).items():
        g["init_sha256." + k] = np.array(v)
    g["param_order"] = np.array([k for k, _ in model.named_parameters()])

    torch.manual_seed(PRUNE_SEED)
    g["keep_idx"] = draw_keep(model)
    model.pre_epoch_processing()
    model.eval()
    with torch.no_grad():
        for tag, adj in (("fwd_sub", model.sub_graph), ("fwd_norm", model.norm_adj)):
            u, i = model.forward(adj)
            G.put(g, tag + "_u", u.numpy())
            G.put(g, tag + "_i", i.numpy())

    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED); torch.manual_seed(BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    g["batch"] = batch.numpy().copy()
    spy = MaskSpy(model.dropoutf)
    model.train()
    for p, rw in REG_CASES.items():
        model.reg_weight = rw
        spy.masks = []
        torch.manual_seed(LOSS_SEED)
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(batch.clone())
        loss.backward()
        assert len(spy.masks) == 4
        if "masks" not in g:
            g["masks"] = np.packbits(np.stack(spy.masks), axis=-1)
            g["masks_shape"] = np.array(np.stack(spy.masks).shape, dtype=np.int64)
        assert np.array_equal(np.packbits(np.stack(spy.masks), axis=-1), g["masks"])
        g[p + "loss"] = loss.detach().numpy().reshape(-1).copy()
        g[p + "loss_shape"] = np.array(loss.shape, dtype=np.int64)
        g[p + "reg_weight"] = np.float64(rw)
        for k, prm in model.named_parameters():
            if prm.grad is not None:
                G.put(g, p + "grad." + k, prm.grad.numpy())
        print(f"PGL reg_weight {rw}: loss {float(loss):.8f}")
    model.reg_weight = config["reg_weight"]
    model.zero_grad(set_to_none=True)
    model.eval()
    with torch.no_grad():
        eb = next(iter(valid_data))
        valid_data.pr = 0; valid_data.inter_pr = 0
        g["eval_users"], g["eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
        s = model.full_sort_predict(eb)
        G.put(g, "scores", s.numpy())
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10                                    # trainer.py:304-309
        g["topk50"] = torch.topk(m, 50, dim=-1)[1].numpy().astype(np.int16)
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g["metric_names"] = np.array(list(res.keys()))
    g["metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g["test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)


def dump_trajectory(out, epochs=2):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("PGL", dict(COMMON, **TRAJ_OVER))
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
        random.seed(TRAJ_SEED0 + ep); np.random.seed(TRAJ_SEED0 + ep); torch.manual_seed(TRAJ_SEED0 + ep)
        n0 = len(rec["batches"])
        rec["keep"].append(draw_keep(model))
        model.pre_epoch_processing()
        trainer._train_epoch(train_data, ep)
        trainer.lr_scheduler.step()
        batch_epoch.append(len(rec["batches"]) - n0)
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    g = {"batch_sizes": np.array([b.shape[1] for b in rec["batches"]]), "batches": np.concatenate(rec["batches"], axis=1),
         "batches_per_epoch": np.array(batch_epoch), "losses": np.array(rec["losses"], dtype=np.float64),
         "valid": np.array(rec["valid"], dtype=np.float64), "test": np.array(rec["test"], dtype=np.float64),
         "keep_idx": np.stack(rec["keep"]), "learning_rate": np.float64(config["learning_rate"]),
         "n_steps": np.int64(len(rec["losses"]))}
    g["metric_names"] = np.array(list(trainer.evaluate(valid_data).keys()))
    for k, v in model.state_dict().items():
        G.put(g, "final." + k, v.numpy())
    np.savez_compressed(out, **g)
    print(f"trajectory PGL: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    install_sparsesvd_stub()
    import logging
    logging.disable(logging.CRITICAL)
    tmp = tempfile.mkdtemp(prefix="mmrec_golden_")
    u, i, e, dim, f = synth.SHAPES[make_golden.DATASET]
    graph = synth.named(make_golden.DATASET)
    v, t = synth.make_features(i, f, seed=1)
    g = {}
    data_root = ref_loader.run_dir(os.path.join(tmp, "model"))
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    dump_model(g)
    data_root = ref_loader.run_dir(os.path.join(tmp, "traj"))
    synth.write_dataset(data_root, make_golden.DATASET, graph, v, t)
    dump_trajectory(os.path.join(HERE, "traj_pgl_tiny.npz"))
    out = os.path.join(HERE, "pgl_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
