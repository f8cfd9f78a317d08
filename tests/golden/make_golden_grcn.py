"""Generate GRCN's golden vectors under tests/golden/ by RUNNING THE REFERENCE ITSELF:

    MMREC_REFERENCE_SRC=<MMRec checkout>/src python tests/golden/make_golden_grcn.py

The unmodified model class (`src/models/grcn.py`) runs under `ref_loader.install()` (its `.cuda()` is the identity on the
CPU) with the harness, dataset and fields of make_golden.py, `train_batch_size` 512.  GRCN imports `torch_geometric`,
which the reference pins no version of; `install_grcn_pyg_shim` below restates, from torch_geometric 2.3's source, the
three things the file uses beyond ref_loader's MMGCN shim (which stays as it is, so the other generators reproduce their
files):
  * `MessagePassing.propagate` with the argument convention of its `message`: `x_j` = x[edge_index[0]], `x_i` =
    x[edge_index[1]], `size_i` = the number of target nodes, `edge_index_i` = edge_index[1] (flow `source_to_target`),
    summed at edge_index[1] ('add');
  * `utils.softmax(src, index, num_nodes)`: the per-group max of the detached scores, `exp` of the difference, the
    per-group sum + 1e-16, a division;
  * `utils.dropout_adj(edge_index, p=0)`: its input, no draw.

Recorded (grcn_tiny.npz), per case: the SHA-256 of every initial `state_dict` entry, the parameter order and the torch RNG
state after construction; `full_sort_predict` of the first validation batch before any training (the random `result`);
on one training batch the final convolution's alpha of each modality and the edge weight in the reference's edge order
(`cat(edge_index, edge_index[[1, 0]])`), `forward`'s representation, the loss and every gradient; then, in evaluation,
`full_sort_predict` of the first validation batch (the batch's representation), the trainer's top-50 of it and the
validation and test metrics.  Tensors above 4096 elements are kept as digest and sketch (`golden_io.put`).
Cases: both modalities at n_layers 3 (the config's, no prefix) and 1 (`l1.`), image only (`image.`).
traj_grcn_tiny.npz: two epochs of the reference's Trainer (both modalities, learning rate 0.001: the config's first grid
value, 1, makes Adam's steps chaotic) with its batches, losses and metrics."""
import inspect
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
CASES = {"": ({}, "vt"), "l1.": ({"n_layers": 1}, "vt"), "image.": ({}, "v")}
BATCH_SEED = 7
TRAJ_SEED0 = 11
TRAJ_LR = 0.001


class MessagePassing(torch.nn.Module):
    """torch_geometric 2.3's `MessagePassing` as far as GRCN uses it (module docstring)."""

    def __init__(self, aggr="add", flow="source_to_target", **kwargs):
        super().__init__()
        if aggr != "add" or flow != "source_to_target":
            raise NotImplementedError((aggr, flow))
        self.aggr, self.flow = aggr, flow

    def propagate(self, edge_index, size=None, **kwargs):
        x = kwargs["x"]
        j, i = edge_index[0], edge_index[1]
        size_i = x.size(0) if size is None else size[1]
        avail = {"x_j": lambda: x.index_select(0, j), "x_i": lambda: x.index_select(0, i), "size_i": lambda: size_i,
                 "edge_index_i": lambda: i, "edge_index_j": lambda: j}
        args = {name: avail[name]() for name in inspect.signature(self.message).parameters}
        msg = self.message(**args)
        out = torch.zeros(size_i, msg.size(1), dtype=msg.dtype, device=msg.device).index_add_(0, i, msg)
        return self.update(out)

    def message(self, x_j):
        return x_j

    def update(self, aggr_out):
        return aggr_out


def softmax(src, index, num_nodes=None):
    """torch_geometric 2.3's `utils.softmax` for a 1-D `src` grouped by `index`."""
    n = int(index.max()) + 1 if num_nodes is None else num_nodes
    src_max = torch.zeros(n, dtype=src.dtype, device=src.device).scatter_reduce_(0, index, src.detach(), "amax", include_self=False)
    out = (src - src_max.index_select(0, index)).exp()
    out_sum = torch.zeros(n, dtype=src.dtype, device=src.device).index_add_(0, index, out) + 1e-16
    return out / out_sum.index_select(0, index)


def dropout_adj(edge_index, edge_attr=None, p=0.5, force_undirected=False, num_nodes=None, training=True):
    if p != 0 and training:
        raise NotImplementedError("dropout_adj with p > 0")
    return edge_index, edge_attr


def install_grcn_pyg_shim():
    pyg = types.ModuleType("torch_geometric")
    nn_m, conv_m, utils_m = (types.ModuleType("torch_geometric." + n) for n in ("nn", "nn.conv", "utils"))
    conv_m.MessagePassing = MessagePassing
    utils_m.softmax, utils_m.dropout_adj = softmax, dropout_adj
    utils_m.remove_self_loops = lambda edge_index, edge_attr=None: (edge_index[:, edge_index[0] != edge_index[1]], edge_attr)
    utils_m.add_self_loops = lambda edge_index, num_nodes=None: (torch.cat([edge_index, torch.arange(num_nodes).repeat(2, 1)], 1), None)
    nn_m.conv, pyg.nn, pyg.utils = conv_m, nn_m, utils_m
    for name, m in (("torch_geometric", pyg), ("torch_geometric.nn", nn_m), ("torch_geometric.nn.conv", conv_m),
                    ("torch_geometric.utils", utils_m)):
        sys.modules[name] = m


def grads(model):
    return {k: p.grad.numpy().copy() for k, p in model.named_parameters() if p.grad is not None}


def dump_model(g, prefix, overrides):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("GRCN", dict(COMMON, **overrides))
    p = prefix
    G.put_sha(g, p + "rng_after_init", torch.get_rng_state().numpy())
    if not prefix:
        inter = train_data.inter_matrix(form="coo")
        g["inter_row"], g["inter_col"] = inter.row.astype(np.int64), inter.col.astype(np.int64)
        g["n_users"], g["n_items"] = np.int64(model.n_users), np.int64(model.n_items)
        for k in ("embedding_size", "latent_embedding", "reg_weight", "learning_rate", "train_batch_size"):
            g["cfg_" + k] = np.float64(config[k])
    g[p + "cfg_n_layers"] = np.int64(config["n_layers"])
    for k, v in G.init_digests(model).items():
        g[p + "init_sha256." + k] = np.array(v)
    g[p + "param_order"] = np.array([k for k, _ in model.named_parameters()])

    eb = next(iter(valid_data))
    valid_data.pr = 0; valid_data.inter_pr = 0
    g[p + "eval_users"], g[p + "eval_mask"] = eb[0].numpy().copy(), eb[1].numpy().copy()
    model.eval()
    with torch.no_grad():
        G.put(g, p + "pre.scores", model.full_sort_predict(eb).numpy())

    random.seed(BATCH_SEED); np.random.seed(BATCH_SEED); torch.manual_seed(BATCH_SEED)
    batch = next(iter(train_data))
    train_data.pr = 0
    seen = {}
    orig_id = model.id_gcn.forward

    def spy_id(edge_index, weight):
        seen["weight"] = weight.detach().numpy().reshape(-1).copy()
        return orig_id(edge_index, weight)
    model.id_gcn.forward = spy_id
    model.train()
    g[p + "batch"] = batch.numpy().copy()
    model.zero_grad(set_to_none=True)
    loss = model.calculate_loss(batch.clone())
    del model.id_gcn.forward
    G.put(g, p + "alpha_v", model.v_gcn.conv_embed_1.alpha.detach().numpy().copy(), whole=True)
    if model.t_feat is not None:
        G.put(g, p + "alpha_t", model.t_gcn.conv_embed_1.alpha.detach().numpy().copy(), whole=True)
    G.put(g, p + "weight", seen["weight"], whole=True)
    G.put(g, p + "representation", model.result.detach().numpy())
    loss.backward()
    g[p + "loss"] = loss.detach().numpy().reshape(-1).copy()
    g[p + "loss_shape"] = np.array(loss.shape, dtype=np.int64)
    for k, v in grads(model).items():
        G.put(g, p + "grad." + k, v)
    model.zero_grad(set_to_none=True)
    model.eval()
    with torch.no_grad():
        s = model.full_sort_predict(eb)
        G.put(g, p + "scores", s.numpy())
        m = s.clone()
        m[eb[1][0], eb[1][1]] = -1e10                                # trainer.py:304-309
        g[p + "topk50"] = torch.topk(m, 50, dim=-1)[1].numpy().astype(np.int16)
    trainer = Trainer(config, model)
    res = trainer.evaluate(valid_data)
    g[p + "metric_names"] = np.array(list(res.keys()))
    g[p + "metric_values"] = np.array([res[k] for k in res], dtype=np.float64)
    g[p + "test_metric_values"] = np.array([v for v in trainer.evaluate(test_data, is_test=True).values()], dtype=np.float64)
    print(f"GRCN{' ' + prefix if prefix else ''}: loss {float(g[p + 'loss'][0]):.6f}")


def dump_trajectory(out, epochs=2):
    from common.trainer import Trainer
    config, train_data, valid_data, test_data, model = make_golden.build("GRCN", dict(COMMON))
    config["epochs"] = epochs
    config["learning_rate"] = TRAJ_LR
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
        model.pre_epoch_processing()
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
    print(f"trajectory GRCN: {len(rec['losses'])} batches, loss {rec['losses'][0]:.6f} -> {rec['losses'][-1]:.6f}")


def main():
    torch.set_num_threads(1)
    ref_loader.install()
    install_grcn_pyg_shim()
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
            dump_trajectory(os.path.join(HERE, "traj_grcn_tiny.npz"))
    out = os.path.join(HERE, "grcn_tiny.npz")
    np.savez_compressed(out, **g)
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
