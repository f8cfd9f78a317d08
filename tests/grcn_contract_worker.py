"""Worker of tests/test_grcn_contract.py: GRCN (`mmrec_b200.models.grcn`) under the harness of tests/contract.py, with
`install_cpu_ops`'s CPU stand-ins plus three for GRCN: the attention graph as its COO in `graph.grcn_edge_order`'s order,
`ops.edge_attention` as PyG's gathers, grouped softmax and `index_add_`, and `ops.spmm_values` as a gather and
`index_add_`.  Against tests/golden/grcn_tiny.npz / traj_grcn_tiny.npz recorded from the reference's class."""
import sys

import torch

import contract as C
import golden_io as G
from make_golden_grcn import CASES, TRAJ_LR, softmax


class _AttnGraph:
    """What GRCN reads of its attention CSR: the entries in CSR order."""

    def __init__(self, rows, cols, n):
        self.rows, self.cols, self.n_rows, self.n_cols = rows, cols, n, n
        self.colidx, self.nnz = cols, rows.numel()


def install():
    from mmrec_b200 import graph, ops

    def build_grcn_adj(inter, n_users, n_items, device):
        rows, cols, order = graph.grcn_edge_order(inter.row, inter.col, n_users, n_items)
        return _AttnGraph(torch.from_numpy(rows), torch.from_numpy(cols), n_users + n_items), torch.from_numpy(order)
    graph.build_grcn_adj = build_grcn_adj

    def edge_attention(A, X, base=None):
        alpha = softmax((X[A.rows] * X[A.cols]).sum(-1), A.rows, num_nodes=A.n_rows)
        Y = torch.zeros_like(X).index_add_(0, A.rows, X[A.cols] * alpha.view(-1, 1))
        return (Y if base is None else base + Y), alpha
    ops.edge_attention = edge_attention
    ops.spmm_values = lambda A, vals, X: torch.zeros_like(X).index_add_(0, A.rows, X[A.cols] * vals.view(-1, 1))


def main_model(p=""):
    over, mods = CASES[p]
    h = C.build("GRCN", mods, over=dict(over), install=install)
    model, sub = h.model, C.case(C.load("grcn_tiny.npz"), p, CASES)
    out = {"init_identical": C.check_init(model, sub)}
    out["pre_score_rel"] = G.rel(sub, "pre.scores", C.predict(model, sub))
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(sub["batch"]))
    out["representation_rel"] = G.rel(sub, "representation", model.result.detach().numpy())
    loss.backward()
    out["grad_keys"], out["grad_rel"] = C.check_grads(model, sub)
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]), "loss_shape": list(loss.shape)})
    model.zero_grad()
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, sub))
    out.update(C.check_metrics(h, sub))
    C.emit(out)


def main_traj():
    h = C.build("GRCN", after={"epochs": 2, "learning_rate": TRAJ_LR}, install=install)
    C.emit(C.replay_trajectory(h, C.load("traj_grcn_tiny.npz")))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    {"traj": main_traj, "l1": lambda: main_model("l1."), "image": lambda: main_model("image.")}.get(arg, main_model)()
