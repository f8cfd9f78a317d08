"""Worker of tests/test_dragon_contract.py: DRAGON (`mmrec_b200.models.dragon`) under the harness of tests/contract.py,
with `install_cpu_ops`'s CPU stand-ins plus `contract.propagate_sum`, against tests/golden/dragon_tiny.npz /
traj_dragon_tiny.npz recorded from the reference's class.  The dataset's `user_graph_dict.npy` is written by
`synth.write_user_graph_dict`."""
import sys

import numpy as np
import torch

import contract as C
import dualgnn_golden as D
import golden_io as G
from make_golden_dragon import CASES

AFTER = {"user_graph_dict_file": "user_graph_dict.npy"}


def install():
    from mmrec_b200 import ops
    ops.propagate_sum = C.propagate_sum


def user_rep(model):
    """`user_rep` before the user graph, from the towers' outputs the forward kept (`v_rep` / `t_rep`, dragon.py:231-243)."""
    U = model.n_users
    if model.v_rep is not None and model.t_rep is not None:
        w = model.weight_u.detach()
        return torch.cat((model.v_rep[:U, :, 0] * w[:, 0], model.t_rep[:U, :, 0] * w[:, 1]), dim=1).detach()
    return (model.t_rep if model.t_rep is not None else model.v_rep)[:U].detach()


def main_model(p=""):
    over, text_only = CASES[p]
    h = C.build("DRAGON", "t" if text_only else "vt", user_graph=True, over={k: [v] for k, v in over.items()}, after=AFTER,
                install=install)
    model, sub = h.model, C.case(C.load("dragon_tiny.npz"), p)
    out = {"init_identical": C.check_init(model, sub) and G.sha256_tagged(model.result_embed.numpy()) == str(sub["result_embed0_sha256"]),
           "has_v_gcn": hasattr(model, "v_gcn")}
    model.eval()
    with torch.no_grad():
        s0 = model.full_sort_predict([torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])])
    out["scores0_equal"] = bool(s0.dtype == torch.float64 and G.equal(sub, "scores0", s0.numpy()))
    np.random.seed(D.SAMPLE_SEED)
    model.pre_epoch_processing()
    out["sample_equal"] = bool(G.equal(sub, "sample_idx", model.epoch_user_graph.numpy())
                               and G.equal(sub, "sample_w", model.user_weight_matrix.numpy()))
    model.train()
    model.zero_grad()
    b = torch.from_numpy(sub["batch"]).clone()
    loss = model.calculate_loss(b)
    out["batch_after_equal"] = bool(np.array_equal(b.numpy(), sub["batch_after"]))
    out["user_rep_rel"] = G.rel(sub, "user_rep", user_rep(model).numpy())
    out["result_embed_rel"] = G.rel(sub, "result_embed", model.result_embed.detach().numpy())
    loss.backward()
    out["grad_keys"], out["grad_rel"] = C.check_grads(model, sub)
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0])})
    model.zero_grad()
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, sub))
    out.update(C.check_metrics(h, sub))
    C.emit(out)


def main_traj():
    h = C.build("DRAGON", user_graph=True, after=dict(AFTER, epochs=2), install=install)
    gold = C.load("traj_dragon_tiny.npz")
    C.emit(C.replay_trajectory(h, gold, lambda ep: np.random.seed(int(gold["epoch_seed0"]) + ep)))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    {"traj": main_traj, "text": lambda: main_model("text."), "mean": lambda: main_model("mean.")}.get(arg, main_model)()
