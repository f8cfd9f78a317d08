"""The harness of the contract workers (tests/*_contract_worker.py), each run in its own process because the kernels behind
`mmrec_b200.ops` are patched.

INTEGRATION.md section 2 claims that the model classes of `mmrec_b200.models` are drop-ins under the reference's
`quick_start` / `Trainer` / dataloaders.  The workers check the claim without a GPU: `build` makes a Config, RecDataset,
TrainDataLoader, EvalDataLoader and Trainer exactly as `src/utils/quick_start.py:26-74` makes them, the model class is OURS,
and the kernels behind `mmrec_b200.ops` are replaced by oracle-backed CPU stand-ins (test infrastructure: the product has no
CPU path).  The harness is the package's own restatement of the reference's (`mmrec_b200.utils`,
`mmrec_b200.common.trainer`, taking the reference's dense evaluation route); with MMREC_REFERENCE_SRC set to the `src/` of an
unmodified enoche/MMRec checkout it is the reference's own code.  Either way the results must equal the golden files
recorded from the reference (tests/golden/).

A worker prints one `CONTRACT <json>` line (`emit`); the tests run it with `run` and assert on the fields."""
import importlib
import json
import os
import subprocess
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
for _p in (GOLDEN, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import golden_io as G  # noqa: E402

BATCHES = {"eval_batch_size": 128, "train_batch_size": 512}


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


def propagate_sum(A, ego, n_layers):
    """Stand-in for ops.propagate_sum: the reference's `h = A x`, `h_1 = A h`, `(h + x) + h_1` (dualgnn.py:314)."""
    out, x = ego, ego
    for _ in range(n_layers):
        x = torch.sparse.mm(A.t_, x)
        out = x + out if out is ego else out + x
    return out


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


def build(name, mods="vt", user_graph=False, over=None, batches=BATCHES, after=None, install=None):
    """OUR class `name` under the harness on the `tiny` dataset, built as src/utils/quick_start.py:26-74 builds it.

    `mods`: the feature tables written ("v" image, "t" text); `user_graph`: also write DualGNN's `user_graph_dict.npy`;
    `over`: config overrides (the reference's list form for hyper-parameters) applied with `batches` before the lists are
    flattened; `after`: config keys set after flattening; `install`: the model's own stand-ins, installed after
    `install_cpu_ops`.  The order -- init_seed, pretrain_setup, stand-ins, construction -- is the reference's: the initial
    weights and the RNG state after construction are compared bit for bit.  Torch runs on one thread, so that every run
    sums in the same order.  Returns config, model, train_data, valid_data, test_data and the Trainer class."""
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v if "v" in mods else None, t if "t" in mods else None)
    if user_graph:
        synth.write_user_graph_dict(data, "tiny", g)
    config = Config(name, "tiny", dict({"gpu_id": 0, "use_gpu": False}, **batches, **(over or {}), **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    for k, val in (after or {}).items():
        config[k] = val
    dataset = RecDataset(config)
    str(dataset)                                                    # (the reference computes inter_num / user_num in __str__)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    install_cpu_ops()
    if install:
        install()
    cls = getattr(importlib.import_module("mmrec_b200.models." + name.lower()), name)
    model = cls(config, train_data).to(config["device"])
    return SimpleNamespace(config=config, model=model, train_data=train_data, valid_data=valid_data, test_data=test_data,
                           Trainer=Trainer)


def load(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=True)


def case(gold, prefix="", prefixes=()):
    """The fields of the case recorded under `prefix`, the prefix stripped: the keys that start with it and with none of
    the longer `prefixes` of the other cases in the file (the default case "" would otherwise take theirs too)."""
    longer = [q for q in prefixes if len(q) > len(prefix)]
    return {k[len(prefix):]: gold[k] for k in map(str, gold.files)
            if k.startswith(prefix) and not any(k.startswith(q) for q in longer)}


def check_init(model, sub, plain=None) -> bool:
    """Bit for bit: every initial state's digest (`init_sha256.*`), the parameter order, and, where the file recorded it,
    torch's RNG state right after construction (which also pins how many draws construction took)."""
    ok = not G.same_init(model, sub, plain) and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]
    if "rng_after_init.sha256" in sub:
        ok = ok and G.equal(sub, "rng_after_init", torch.get_rng_state().numpy())
    return bool(ok)


def check_grads(model, sub, prefix="grad."):
    """(the parameters that got a gradient are exactly the recorded ones, {name: rel of its gradient})."""
    named = dict(model.named_parameters())
    keys = [k[len(prefix):] for k in G.recorded(sub, prefix)]
    return (sorted(k for k, q in named.items() if q.grad is not None) == keys,
            {k: G.rel(sub, prefix + k, named[k].grad.numpy()) for k in keys})


def predict(model, sub):
    """`full_sort_predict` in eval mode on the recorded evaluation batch, as a numpy array."""
    model.eval()
    with torch.no_grad():
        return model.full_sort_predict([torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])]).numpy()


def check_metrics(h, sub) -> dict:
    """`Trainer.evaluate` on the valid and (where the file recorded them) test loaders, and the recorded metrics by name."""
    trainer = h.Trainer(h.config, h.model)
    names = [str(x) for x in sub["metric_names"]]
    out = {}
    for part, data, key in (("valid", h.valid_data, "metric_values"), ("test", h.test_data, "test_metric_values")):
        if key in sub:
            out[part] = {k: float(v) for k, v in trainer.evaluate(data, is_test=part == "test").items()}
            out["want_" + part] = dict(zip(names, [float(x) for x in sub[key]]))
    return out


def recorded_batches(gold):
    """The trajectory's recorded batches, per epoch."""
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    batches = gold["batches"]
    return [[torch.from_numpy(batches[:, offs[b]:offs[b + 1]].copy()) for b in range(first[ep], first[ep + 1])]
            for ep in range(len(gold["batches_per_epoch"]))]


def replay_trajectory(h, gold, before_epoch=None, epochs=None):
    """Two epochs of `Trainer._train_epoch` (its Adam, its scheduler) on `epochs` (default: the recorded batches), each
    followed by the valid and test evaluations; `before_epoch(ep)` runs before the epoch's `pre_epoch_processing`.  Every
    batch's loss and the per-epoch metrics are compared with the recorded trajectory."""
    model, trainer = h.model, h.Trainer(h.config, h.model)
    losses, valid, test = [], [], []
    orig = model.calculate_loss

    def spy(interaction):
        l = orig(interaction)
        losses.append(float(sum(l)) if isinstance(l, tuple) else float(l.detach()))
        return l
    model.calculate_loss = spy
    epochs = recorded_batches(gold) if epochs is None else epochs
    for ep in range(2):
        if before_epoch:
            before_epoch(ep)
        model.pre_epoch_processing()
        trainer._train_epoch(epochs[ep], ep)
        trainer.lr_scheduler.step()
        valid.append(list(trainer.evaluate(h.valid_data).values()))
        test.append(list(trainer.evaluate(h.test_data, is_test=True).values()))
    out = {"n_batches": len(losses), "loss_max_rel": float(np.max(np.abs(np.array(losses) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(valid) - gold["valid"]).max(), np.abs(np.array(test) - gold["test"]).max()))}
    if "n_steps" in gold:
        out["want_batches"] = int(gold["n_steps"])
    return out


def emit(out):
    print("CONTRACT " + json.dumps(out))


def run(worker, arg=None, timeout=900):
    """Run tests/<worker> (with `arg`) in its own process and return the fields of its CONTRACT line."""
    out = subprocess.run([sys.executable, os.path.join(HERE, worker)] + ([] if arg is None else [arg]), capture_output=True,
                         text=True, timeout=timeout)
    lines = [l for l in out.stdout.splitlines() if l.startswith("CONTRACT ")]
    assert out.returncode == 0 and lines, out.stdout[-3000:] + out.stderr[-3000:]
    return json.loads(lines[-1][len("CONTRACT "):])


def assert_metrics(r):
    """The valid and test metrics have the recorded names and values (the evaluator's float64 rounding aside)."""
    assert "want_valid" in r
    for part in [p for p in ("valid", "test") if "want_" + p in r]:
        assert r[part].keys() == r["want_" + part].keys(), (part, sorted(r[part]), sorted(r["want_" + part]))
        for k, v in r["want_" + part].items():
            assert abs(r[part][k] - v) < 1e-9, (part, k, r[part][k], v)
