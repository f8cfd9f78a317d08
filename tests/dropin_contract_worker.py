"""Worker of tests/test_dropin_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

INTEGRATION.md section 2 claims that the model classes of `mmrec_b200.models` are drop-ins under the reference's
`quick_start` / `Trainer` / dataloaders.  This checks the claim without a GPU: a Config, RecDataset, TrainDataLoader,
EvalDataLoader and Trainer are built exactly as `src/utils/quick_start.py:26-74` builds them, the model class is OURS, and the
kernels behind `mmrec_b200.ops` are replaced by oracle-backed CPU stand-ins (test infrastructure: the product has no CPU
path).  The harness is the package's own restatement of the reference's (`mmrec_b200.utils`, `mmrec_b200.common.trainer`,
taking the reference's dense evaluation route); with MMREC_REFERENCE_SRC set to the `src/` of an unmodified enoche/MMRec
checkout it is the reference's own code.  Either way the results must equal the golden files recorded from the reference.  `Trainer.evaluate` (the reference's: full_sort_predict -> in-place mask -> torch.topk -> its own TopKEvaluator) must
return the metrics recorded from the reference's own model, and one `calculate_loss` through `Trainer._train_epoch`'s call
path must return the recorded loss."""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "golden"))


class CpuCSR:
    """Stand-in for ops.CSR: a coalesced torch sparse matrix on the CPU."""

    def __init__(self, t, symmetric=False):
        self.t_, self.n_rows, self.n_cols, self.nnz, self.symmetric = t, t.shape[0], t.shape[1], t._nnz(), symmetric

    @staticmethod
    def from_coo(row, col, val, n_rows, n_cols, sum_duplicates=True, symmetric=False, seg=None, light_max=None):
        val = torch.ones(row.numel(), dtype=torch.float32) if val is None else val.to(torch.float32)
        t = torch.sparse_coo_tensor(torch.stack([row.to(torch.int64), col.to(torch.int64)]), val, (n_rows, n_cols))
        return CpuCSR(t.coalesce() if sum_duplicates else t.coalesce(), symmetric)

    @staticmethod
    def from_torch_sparse(t, symmetric=False):
        return CpuCSR(t.coalesce(), symmetric)

    def coo(self):
        i = self.t_.indices()
        return i[0], i[1], self.t_.values()

    def t(self):
        return self if self.symmetric else CpuCSR(self.t_.t().coalesce())


def install_cpu_ops():
    from oracle import mmrec_oracle as O
    from mmrec_b200 import graph, ops
    ops.CSR = graph.CSR = CpuCSR
    ops.propagate_mean = lambda A, ego, n_layers: O.propagate_mean(A.t_, ego, n_layers)
    ops.spmm = lambda A, X, base=None: torch.sparse.mm(A.t_, X) if base is None else base + torch.sparse.mm(A.t_, X)
    ops.project = lambda table, weight, bias=None, idx=None, l2_normalize=False: O.project(table, weight, bias, idx=idx, l2_normalize=l2_normalize)
    ops.score = lambda u, i, users=None: O.full_sort_scores(u, i, users if users is not None else torch.arange(u.shape[0]))

    def mask_topk(scores, mask, k, item_offset=0):                    # graph._knn, and the trainer's dense route
        if mask is not None:
            scores[mask[0], mask[1] - item_offset] = -1e10                # trainer.py:305-309
        return torch.topk(scores, k, dim=-1)
    ops.mask_topk = mask_topk

    def bipartite_norm(users, items, n_users, n_items, eps=1e-7):
        return O.normalize_adj_m(torch.stack([users, items]), n_users, n_items)
    ops.bipartite_norm = bipartite_norm

    # inference-only entry points (restated from their documented formulas in include/mmrec_b200.h)
    def spmm_raw(A, X, Y=None, acc_in=None, acc_out=None, acc_div=1.0, gate_ref=None, use_plan=True, y_accumulate=False):
        y = torch.sparse.mm(A.t_, X)
        if gate_ref is not None:
            y = torch.nn.functional.cosine_similarity(y, gate_ref, dim=-1).unsqueeze(1) * y
        if acc_out is not None:
            acc_out.copy_(((y if acc_in is None else acc_in + y)) / acc_div)
        if Y is not None:
            Y.copy_(Y + y if y_accumulate else y)
    ops.spmm_raw = spmm_raw

    def gate_rows(x, weight, bias, mul=None, out=None):
        r = torch.sigmoid(torch.nn.functional.linear(x, weight, bias))
        r = r if mul is None else mul * r
        return r if out is None else out.copy_(r)
    ops.gate_rows = gate_rows

    def mgcn_fuse(img, txt, content, q_w, q_b, q_w2, gi_w, gi_b, gt_w, gt_b, want_side=False):
        lin = torch.nn.functional.linear
        att = torch.cat([lin(torch.tanh(lin(img, q_w, q_b)), q_w2), lin(torch.tanh(lin(txt, q_w, q_b)), q_w2)], dim=-1)
        w = torch.softmax(att, dim=-1)
        common = w[:, 0].unsqueeze(1) * img + w[:, 1].unsqueeze(1) * txt
        side = (torch.sigmoid(lin(content, gi_w, gi_b)) * (img - common) + torch.sigmoid(lin(content, gt_w, gt_b)) * (txt - common) + common) / 3
        return (content + side, side) if want_side else content + side
    ops.mgcn_fuse = mgcn_fuse

    def propagate_layergcn(A, ego, n_layers):
        acc, x = torch.zeros_like(ego), ego
        for _ in range(n_layers):
            x = torch.sparse.mm(A.t_, x)
            x = torch.nn.functional.cosine_similarity(x, ego, dim=-1).unsqueeze(1) * x
            acc = acc + x
        return acc
    ops.propagate_layergcn = propagate_layergcn


def harness(tmp):
    """(data directory, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra config keys)."""
    if os.environ.get("MMREC_REFERENCE_SRC"):
        import ref_loader
        ref_loader.install()
        data = ref_loader.run_dir(tmp)
        from utils.configurator import Config
        from utils.dataset import RecDataset
        from utils.dataloader import TrainDataLoader, EvalDataLoader
        from utils.utils import init_seed
        from common.trainer import Trainer
        return data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, {}
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import init_seed
    data = os.path.join(tmp, "data")
    os.makedirs(data, exist_ok=True)
    # the reference's routes: dense full_sort_predict -> mask -> top-k, host evaluator, torch.optim.Adam
    extra = {"data_path": data + "/", "use_fused_topk": False, "device_evaluator": False, "fused_adam": False}
    return data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra


def main():
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    # --- the harness, built as src/utils/quick_start.py:26-74 builds it
    config = Config("FREEDOM", "tiny", dict({"gpu_id": 0, "use_gpu": False, "n_ui_layers": 3}, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    dataset = RecDataset(config)
    str(dataset)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    # --- OUR model class, the way utils.get_model would return it from src/models/freedom.py (INTEGRATION.md section 2)
    install_cpu_ops()
    from mmrec_b200.models.freedom import FREEDOM
    model = FREEDOM(config, train_data).to(config["device"])
    gold = np.load(os.path.join(HERE, "golden", "freedom_tiny.npz"), allow_pickle=True)
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0."))
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in gold["metric_names"]]
    want_valid = dict(zip(names, [float(x) for x in gold["metric_values"]]))
    want_test = dict(zip(names, [float(x) for x in gold["test_metric_values"]]))
    # --- one loss through the call the reference's _train_epoch makes (src/common/trainer.py:147-153), on the recorded batch
    from mmrec_b200 import graph
    model.train()
    model.masked_adj = model.pruner.adj_from_keep(torch.from_numpy(gold["prune_keep_idx"]))
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss = sum(loss) if isinstance(loss, tuple) else loss
    loss.backward()                                                 # autograd-connected to the parameters (the optimiser steps on them)
    has_grads = all(p.grad is not None for p in model.parameters())
    out = {"init_identical": bool(init_identical), "valid": {k: float(v) for k, v in valid.items()}, "want_valid": want_valid,
           "test": {k: float(v) for k, v in test.items()}, "want_test": want_test, "loss": float(loss.item()),
           "want_loss": float(np.asarray(gold["loss"]).sum()), "has_grads": bool(has_grads)}
    print("CONTRACT " + json.dumps(out))


def main_mmgcn():
    """The same for MMGCN: OUR class (no torch_geometric needed) under the harness against
    tests/golden/mmgcn_tiny.npz, the reference's own model code run under a PyG shim (tests/golden/ref_loader.py)."""
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    config = Config("MMGCN", "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    dataset = RecDataset(config)
    str(dataset)                                                    # (the reference computes inter_num / user_num in __str__)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    install_cpu_ops()
    from mmrec_b200.models.mmgcn import MMGCN
    model = MMGCN(config, train_data).to(config["device"])
    gold = np.load(os.path.join(HERE, "golden", "mmgcn_tiny.npz"), allow_pickle=True)
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]] \
        and np.array_equal(model.id_embedding.detach().numpy(), gold["id_embedding"]) \
        and np.array_equal(model.v_gcn.preference.detach().numpy(), gold["v_preference"]) \
        and np.array_equal(model.t_gcn.preference.detach().numpy(), gold["t_preference"])

    def rel(a, b):
        return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / np.linalg.norm(b))
    model.train()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss.backward()
    grad_rel = max(rel(p.grad.numpy(), gold["grad." + k]) for k, p in model.named_parameters() if "grad." + k in gold.files)
    model.eval()
    with torch.no_grad():
        fwd_rel = rel(model.forward().numpy(), gold["fwd"])
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
        score_err = float(np.abs(sc.numpy() - gold["scores"]).max())
    valid = Trainer(config, model).evaluate(valid_data)
    names = [str(x) for x in gold["metric_names"]]
    out = {"init_identical": bool(init_identical), "fwd_rel": fwd_rel, "loss": float(loss.item()), "want_loss": float(gold["loss"][0]),
           "grad_rel": grad_rel, "score_err": score_err, "valid": {k: float(v) for k, v in valid.items()},
           "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]]))}
    print("CONTRACT " + json.dumps(out))


def main_model(name):
    """BM3 / MGCN / LightGCN / LayerGCN: our class under the harness against the golden file of the reference's
    own class -- initial weights, `forward`, the loss on the recorded batch WITH the reference's RNG draws (BM3's always-on
    dropout: same `torch.manual_seed(4321)` stream as tests/golden/make_golden.py), first-batch scores, `Trainer.evaluate`."""
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    over = {"BM3": {}, "MGCN": {}, "LightGCN": {"n_layers": [3]}, "LayerGCN": {"dropout": [0.1]}}[name]
    config = Config(name, "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **over, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    dataset = RecDataset(config)
    str(dataset)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    install_cpu_ops()
    import importlib
    cls = getattr(importlib.import_module("mmrec_b200.models." + name.lower()), name)
    model = cls(config, train_data).to(config["device"])
    gold = np.load(os.path.join(HERE, "golden", name.lower() + "_tiny.npz"), allow_pickle=True)
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]

    def rel(a, b):
        return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / max(np.linalg.norm(b), 1e-30))
    model.eval()
    with torch.no_grad():
        if name == "MGCN":
            fu, fi = model.forward(model.norm_adj)                   # no autograd: the gate / fuse / stacked-table route (a5b)
        elif name == "LayerGCN":
            model.forward_adj = model.norm_adj_matrix
            fu, fi = model.forward()
        else:
            fu, fi = model.forward()
    fwd_rel = max(rel(fu.numpy(), gold["fwd_u"]), rel(fi.numpy(), gold["fwd_i"]))
    model.train()
    torch.manual_seed(1234)
    if name == "LayerGCN":
        model.masked_adj = model.pruner.adj_from_keep(torch.from_numpy(gold["prune_keep_idx"]))
    torch.manual_seed(4321)                                          # BM3's F.dropout draws, as in make_golden.py
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss = sum(loss) if isinstance(loss, tuple) else loss
    loss.backward()
    named = dict(model.named_parameters())
    gmax = max(float(np.abs(gold[k]).max()) for k in gold.files if k.startswith("grad."))
    grad_ok = all(np.linalg.norm(named[k[5:]].grad.numpy().astype(np.float64) - gold[k]) < 1e-4 * np.linalg.norm(gold[k]) + 1e-7 * gmax * np.sqrt(gold[k].size)
                  for k in gold.files if k.startswith("grad."))
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
    score_err = float(np.abs(sc.numpy() - gold["scores"]).max() / np.abs(gold["scores"]).max())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in gold["metric_names"]]
    out = {"model": name, "init_identical": bool(init_identical), "fwd_rel": fwd_rel, "loss": float(loss.item()),
           "want_loss": float(np.asarray(gold["loss"]).sum()), "grad_ok": bool(grad_ok), "score_err": score_err,
           "valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
           "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))}
    print("CONTRACT " + json.dumps(out))


def main_traj(key):
    """Two epochs of the training loop (`Trainer._train_epoch`, its Adam, its scheduler, its dataloader's shuffling and
    negative sampling) driving OUR class, against the trajectory the reference's class produced
    (tests/golden/traj_*_tiny.npz: every batch, every batch loss, per-epoch metrics)."""
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    # key -> (model class, overrides of make_golden.py's dump_trajectory call, golden file)
    name, over, gfile = {"LightGCN": ("LightGCN", {"n_layers": [2], "reg_weight": [1e-4]}, "traj_lightgcn_tiny.npz"),
                         "FREEDOM": ("FREEDOM", {"dropout": [0.0], "reg_weight": [1e-3]}, "traj_freedom_tiny.npz"),
                         "FREEDOM-prune": ("FREEDOM", {"dropout": [0.8], "reg_weight": [1e-3]}, "traj_freedom_prune_tiny.npz"),
                         "LayerGCN": ("LayerGCN", {"dropout": [0.1]}, "traj_layergcn_tiny.npz"),
                         "BM3": ("BM3", {}, "traj_bm3_tiny.npz"),
                         "MGCN": ("MGCN", {}, "traj_mgcn_tiny.npz")}[key]
    config = Config(name, "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **over, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    config["epochs"] = 2
    dataset = RecDataset(config)
    str(dataset)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    install_cpu_ops()
    import importlib
    model = getattr(importlib.import_module("mmrec_b200.models." + name.lower()), name)(config, train_data).to(config["device"])
    gold = np.load(os.path.join(os.environ.get("MMREC_TRAJ_DIR", os.path.join(HERE, "golden")), gfile), allow_pickle=True)
    trainer = Trainer(config, model)
    rec = {"batches": [], "losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        rec["batches"].append(interaction.numpy().copy())
        l = orig(interaction)
        rec["losses"].append(float(sum(l)) if isinstance(l, tuple) else float(l))
        return l
    model.calculate_loss = spy
    # The reference's own loader reproduces its shuffling and negative-sampling stream, so its batches are compared.  The
    # package's loader keeps the reference's batch format but draws its own stream (vectorised sampling), so with the
    # package harness the recorded batches are replayed and every loss and metric is compared.
    replay = not os.environ.get("MMREC_REFERENCE_SRC")
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    recorded = [[torch.from_numpy(gold["batches"][:, offs[b]:offs[b + 1]]) for b in range(first[ep], first[ep + 1])]
                for ep in range(len(gold["batches_per_epoch"]))]
    # LayerGCN's uniform pruning draws from Python's `random`, the stream the reference's loader samples negatives from:
    # its state at the start of each epoch is recorded from the reference run (MMREC_RECORD_DIR) and restored in replay.
    import random
    state_file = os.path.join(HERE, "golden", "traj_%s_tiny_pyrandom.npz" % key.lower())
    states = []
    for ep in range(2):
        if replay and os.path.isfile(state_file):
            st = np.load(state_file)["state%d" % ep]
            random.setstate((int(st[0]), tuple(int(x) for x in st[1:-1]), None))
        states.append(np.array([random.getstate()[0]] + list(random.getstate()[1]) + [0], dtype=np.int64))
        model.pre_epoch_processing()
        trainer._train_epoch(recorded[ep] if replay else train_data, ep)
        trainer.lr_scheduler.step()
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data).values()))
    if not replay and os.environ.get("MMREC_RECORD_DIR"):
        np.savez(os.path.join(os.environ["MMREC_RECORD_DIR"], "traj_%s_tiny_pyrandom.npz" % key.lower()),
                 **{"state%d" % ep: st for ep, st in enumerate(states)})
    batches = np.concatenate(rec["batches"], axis=1)
    out = {"model": name, "batches": "recorded, replayed" if replay else "drawn by the reference's loader",
           "same_batches": bool(batches.shape == gold["batches"].shape and np.array_equal(batches, gold["batches"])),
           "n_batches": len(rec["losses"]), "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max())),
           "first_loss": rec["losses"][0], "last_loss": rec["losses"][-1], "want_last_loss": float(gold["losses"][-1])}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    if arg.startswith("traj:"):
        main_traj(arg[5:]); sys.exit(0)
    main_mmgcn() if arg == "mmgcn" else (main_model(arg) if arg else main())
