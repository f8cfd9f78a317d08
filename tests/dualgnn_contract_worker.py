"""Worker of tests/test_dualgnn_contract.py: DualGNN (`mmrec_b200.models.dualgnn`) under the harness of tests/contract.py,
with `install_cpu_ops`'s CPU stand-ins plus `contract.propagate_sum`, against tests/golden/dualgnn_tiny.npz /
traj_dualgnn_tiny.npz recorded from the reference's class.  The dataset's `user_graph_dict.npy` is written by
`synth.write_user_graph_dict`."""
import sys

import numpy as np
import torch

import contract as C
import dualgnn_golden as D
import golden_io as G

AFTER = {"user_graph_dict_file": "user_graph_dict.npy"}


def install():
    from mmrec_b200 import ops
    ops.propagate_sum = C.propagate_sum


def main_model(p=""):
    h = C.build("DualGNN", "t" if p == "text." else "vt", user_graph=True, after=AFTER, install=install)
    model, sub = h.model, C.case(C.load("dualgnn_tiny.npz"), p)
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
    seen = {}
    orig = model.user_graph.forward

    def spy(features, user_graph, user_matrix=None, base=None):
        seen["user_rep"] = features.detach().numpy().copy()
        return orig(features, user_graph, user_matrix, base=base)
    model.user_graph.forward = spy
    model.train()
    model.zero_grad()
    b = torch.from_numpy(sub["batch"]).clone()
    loss = model.calculate_loss(b)
    out["batch_after_equal"] = bool(np.array_equal(b.numpy(), sub["batch_after"]))
    out["rep_rel"] = {n: G.rel(sub, n, getattr(model, n).detach().squeeze(2).numpy()) for n in ("v_rep", "t_rep")
                      if n + ".sha256" in sub}
    out["user_rep_rel"] = G.rel(sub, "user_rep", seen["user_rep"])
    out["result_embed_rel"] = G.rel(sub, "result_embed", model.result_embed.detach().numpy())
    loss.backward()
    out["grad_keys"], out["grad_rel"] = C.check_grads(model, sub)
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0])})
    model.zero_grad()
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, sub))
    out.update(C.check_metrics(h, sub))
    C.emit(out)


def main_traj():
    h = C.build("DualGNN", user_graph=True, after=dict(AFTER, epochs=2), install=install)
    gold = C.load("traj_dualgnn_tiny.npz")
    C.emit(C.replay_trajectory(h, gold, lambda ep: np.random.seed(int(gold["epoch_seed0"]) + ep)))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    {"traj": main_traj, "text": lambda: main_model("text.")}.get(arg, main_model)()
