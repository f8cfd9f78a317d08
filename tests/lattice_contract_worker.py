"""Worker of tests/test_lattice_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

LATTICE (`mmrec_b200.models.lattice`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start
builds it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by
`install_cpu_ops`'s CPU stand-ins plus torch restatements of the learned graph's operators (`ops.sddmm`,
`ops.csr_sym_norm`, `ops.spmm_values` and the pattern CSR the model builds directly), against tests/golden/lattice_tiny.npz
and traj_lattice_tiny.npz recorded from the reference's class."""
import copy
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import dualgnn_golden as G  # noqa: E402
import selfcf_golden  # noqa: E402
from dropin_contract_worker import CpuCSR, harness, install_cpu_ops  # noqa: E402
from make_golden_lattice import CASES  # noqa: E402


class LatticeCpuCSR(CpuCSR):
    """`CpuCSR`, plus what LATTICE reads of `ops.CSR`: the constructor from (rowptr, colidx, vals), `vals` and
    `with_values`.  Entries are kept in CSR order (row, then stored column)."""

    def __init__(self, *a, **k):
        if isinstance(a[0], torch.Tensor):
            super().__init__(*a, **k)
            i = self.t_.indices()
            self.row, self.col, self.vals = i[0], i[1], self.t_.values()
            return
        n_rows, n_cols, rowptr, colidx, vals, nnz = a[:6]
        self.n_rows, self.n_cols, self.nnz, self.symmetric = int(n_rows), int(n_cols), int(nnz), False
        self.row = torch.repeat_interleave(torch.arange(self.n_rows), (rowptr[1:] - rowptr[:-1]).to(torch.int64))
        self.col, self.vals = colidx[:self.nnz].to(torch.int64), vals[:self.nnz]

    @staticmethod
    def from_coo(*a, **k):
        c = CpuCSR.from_coo(*a, **k)
        return LatticeCpuCSR(c.t_, c.symmetric)

    def t(self):
        return self if self.symmetric else LatticeCpuCSR(self.t_.t().coalesce())

    def with_values(self, vals):
        out = copy.copy(self)
        out.vals = vals
        return out


def install():
    install_cpu_ops()
    from mmrec_b200 import graph, ops
    ops.CSR = graph.CSR = LatticeCpuCSR
    ops.sddmm = lambda A, P, Q: (P[A.row] * Q[A.col]).sum(1)

    def csr_sym_norm(A, vals):
        rowsum = torch.zeros(A.n_rows, dtype=vals.dtype).index_add(0, A.row, vals)
        d = rowsum.pow(-0.5)
        d = d.masked_fill(torch.isinf(d), 0.0)
        return (d[A.row] * vals) * d[A.col]
    ops.csr_sym_norm = csr_sym_norm
    ops.spmm_values = lambda A, vals, X: torch.zeros(A.n_rows, X.shape[1], dtype=X.dtype).index_add(0, A.row, vals.unsqueeze(1) * X[A.col])


def _data(mods):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, *rest = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v if "v" in mods else None, t if "t" in mods else None)
    return rest


def _build(rest, over, epochs=None):
    Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = rest
    config = Config("LATTICE", "tiny", dict({"gpu_id": 0, "use_gpu": False, "train_batch_size": 512}, **over, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    if epochs:
        config["epochs"] = epochs
    dataset = RecDataset(config)
    str(dataset)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    from mmrec_b200.models.lattice import LATTICE
    model = LATTICE(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def _sub(gold, p):
    keys = [str(k) for k in gold.files]
    if p:
        return {k[len(p):]: gold[k] for k in keys if k.startswith(p)}
    return {k: gold[k] for k in keys if not any(k.startswith(q) for q in CASES if q)}


def check_case(rest, p, gold):
    sub = _sub(gold, p)
    config, model, valid_data, test_data, Trainer = _build(rest, dict(CASES[p][0]))
    init = {k[len("init_sha256."):]: str(v) for k, v in sub.items() if k.startswith("init_sha256.")}
    out = {"init_identical": selfcf_golden.init_digests(model) == init
           and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]}
    model.train()
    model.pre_epoch_processing()
    named = dict(model.named_parameters())
    out["grad_rel"], out["loss_rel"], out["grad_keys"] = 0.0, 0.0, True
    for tag in ("build.", "plain."):
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(torch.from_numpy(sub[tag + "batch"]))
        loss.backward()
        want = float(sub[tag + "loss"][0])
        out["loss_rel"] = max(out["loss_rel"], abs(float(loss.item()) - want) / abs(want))
        grads = [k[len(tag + "grad."):] for k in G.recorded(sub, tag + "grad.")]
        if tag == "plain." and not grads:                               # recorded for the first case only
            continue
        out["grad_keys"] &= sorted(k for k, q in named.items() if q.grad is not None) == sorted(grads)
        out["grad_rel"] = max([out["grad_rel"]] + [G.rel(sub, tag + "grad." + k, named[k].grad.numpy()) for k in grads])
    model.zero_grad(set_to_none=True)
    model.eval()
    eb = [torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])]
    with torch.no_grad():
        out["score_rel"] = G.rel(sub, "scores", model.full_sort_predict(eb).numpy())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in sub["metric_names"]]
    out["metric_max_abs"] = max(max(abs(valid[k] - w) for k, w in zip(names, sub["metric_values"])),
                                max(abs(test[k] - w) for k, w in zip(names, sub["test_metric_values"])))
    return out


def main_model():
    gold = np.load(os.path.join(HERE, "golden", "lattice_tiny.npz"), allow_pickle=True)
    install()
    res = {}
    for p, (_, mods) in CASES.items():
        res[p or "default"] = check_case(_data(mods), p, gold)
    print("CONTRACT " + json.dumps(res))


def main_traj():
    gold = np.load(os.path.join(HERE, "golden", "traj_lattice_tiny.npz"), allow_pickle=True)
    install()
    config, model, valid_data, test_data, Trainer = _build(_data("vt"), {}, epochs=2)
    trainer = Trainer(config, model)
    rec = {"losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        l = orig(interaction)
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    recorded = [[torch.from_numpy(gold["batches"][:, offs[b]:offs[b + 1]].copy()) for b in range(first[ep], first[ep + 1])]
                for ep in range(len(gold["batches_per_epoch"]))]
    for ep in range(2):
        model.pre_epoch_processing()
        trainer._train_epoch(recorded[ep], ep)
        trainer.lr_scheduler.step()
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    out = {"n_batches": len(rec["losses"]), "want_batches": int(gold["n_steps"]),
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    main_traj() if (sys.argv[1] if len(sys.argv) > 1 else "") == "traj" else main_model()
