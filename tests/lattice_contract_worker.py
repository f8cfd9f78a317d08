"""Worker of tests/test_lattice_contract.py: LATTICE (`mmrec_b200.models.lattice`) under the harness of tests/contract.py,
with `install_cpu_ops`'s CPU stand-ins plus torch restatements of the learned graph's operators (`ops.sddmm`,
`ops.csr_sym_norm`, `ops.spmm_values` and the pattern CSR the model builds directly), against tests/golden/lattice_tiny.npz
and traj_lattice_tiny.npz recorded from the reference's class."""
import copy
import sys

import torch

import contract as C
import golden_io as G
from make_golden_lattice import CASES

BATCHES = {"train_batch_size": 512}


class LatticeCpuCSR(C.CpuCSR):
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
        c = C.CpuCSR.from_coo(*a, **k)
        return LatticeCpuCSR(c.t_, c.symmetric)

    def t(self):
        return self if self.symmetric else LatticeCpuCSR(self.t_.t().coalesce())

    def with_values(self, vals):
        out = copy.copy(self)
        out.vals = vals
        return out


def install():
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


def check_case(p, gold):
    over, mods = CASES[p]
    h = C.build("LATTICE", mods, over=dict(over), batches=BATCHES, install=install)
    model, sub = h.model, C.case(gold, p, CASES)
    out = {"init_identical": C.check_init(model, sub)}
    model.train()
    model.pre_epoch_processing()
    out["grad_rel"], out["loss_rel"], out["grad_keys"] = 0.0, 0.0, True
    for tag in ("build.", "plain."):
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(torch.from_numpy(sub[tag + "batch"]))
        loss.backward()
        want = float(sub[tag + "loss"][0])
        out["loss_rel"] = max(out["loss_rel"], abs(float(loss.item()) - want) / abs(want))
        if tag == "plain." and not G.recorded(sub, tag + "grad."):        # recorded for the first case only
            continue
        keys_ok, rels = C.check_grads(model, sub, tag + "grad.")
        out["grad_keys"] &= keys_ok
        out["grad_rel"] = max([out["grad_rel"]] + list(rels.values()))
    model.zero_grad(set_to_none=True)
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, sub))
    out.update(C.check_metrics(h, sub))
    return out


def main_model():
    gold = C.load("lattice_tiny.npz")
    C.emit({p or "default": check_case(p, gold) for p in CASES})


def main_traj():
    h = C.build("LATTICE", batches=BATCHES, after={"epochs": 2}, install=install)
    C.emit(C.replay_trajectory(h, C.load("traj_lattice_tiny.npz")))


if __name__ == "__main__":
    main_traj() if (sys.argv[1] if len(sys.argv) > 1 else "") == "traj" else main_model()
