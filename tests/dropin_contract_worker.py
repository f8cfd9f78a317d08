"""Worker of tests/test_dropin_contract.py: FREEDOM, MMGCN, BM3, MGCN, LightGCN and LayerGCN under the harness of
tests/contract.py.  `Trainer.evaluate` (the reference's: full_sort_predict -> in-place mask -> torch.topk -> its own
TopKEvaluator) must return the metrics recorded from the reference's own model, and one `calculate_loss` through
`Trainer._train_epoch`'s call path must return the recorded loss."""
import os
import random
import sys

import numpy as np
import torch

import contract as C
import golden_io as G


def main():
    h = C.build("FREEDOM", over={"n_ui_layers": 3}, batches={})
    model, gold = h.model, C.load("freedom_tiny.npz")
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0."))
    out = {"init_identical": bool(init_identical)}
    out.update(C.check_metrics(h, gold))
    # --- one loss through the call the reference's _train_epoch makes (src/common/trainer.py:147-153), on the recorded batch
    model.train()
    model.masked_adj = model.pruner.adj_from_keep(torch.from_numpy(gold["prune_keep_idx"]))
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss = sum(loss) if isinstance(loss, tuple) else loss
    loss.backward()                                                 # autograd-connected to the parameters (the optimiser steps on them)
    out.update({"loss": float(loss.item()), "want_loss": float(np.asarray(gold["loss"]).sum()),
                "has_grads": all(p.grad is not None for p in model.parameters())})
    C.emit(out)


def main_mmgcn():
    """The same for MMGCN: OUR class (no torch_geometric needed) against tests/golden/mmgcn_tiny.npz, the reference's own
    model code run under a PyG shim (tests/golden/ref_loader.py)."""
    h = C.build("MMGCN")
    model, gold = h.model, C.load("mmgcn_tiny.npz")
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]] \
        and np.array_equal(model.id_embedding.detach().numpy(), gold["id_embedding"]) \
        and np.array_equal(model.v_gcn.preference.detach().numpy(), gold["v_preference"]) \
        and np.array_equal(model.t_gcn.preference.detach().numpy(), gold["t_preference"])
    model.train()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss.backward()
    grad_rel = max(G.rel_to(p.grad.numpy(), gold["grad." + k]) for k, p in model.named_parameters() if "grad." + k in gold.files)
    model.eval()
    with torch.no_grad():
        fwd_rel = G.rel_to(model.forward().numpy(), gold["fwd"])
    score_err = float(np.abs(C.predict(model, gold) - gold["scores"]).max())
    out = {"init_identical": bool(init_identical), "fwd_rel": fwd_rel, "loss": float(loss.item()), "want_loss": float(gold["loss"][0]),
           "grad_rel": grad_rel, "score_err": score_err}
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_model(name):
    """BM3 / MGCN / LightGCN / LayerGCN: our class against the golden file of the reference's own class -- initial weights,
    `forward`, the loss on the recorded batch WITH the reference's RNG draws (BM3's always-on dropout: same
    `torch.manual_seed(4321)` stream as tests/golden/make_golden.py), first-batch scores, `Trainer.evaluate`."""
    over = {"BM3": {}, "MGCN": {}, "LightGCN": {"n_layers": [3]}, "LayerGCN": {"dropout": [0.1]}}[name]
    h = C.build(name, over=over)
    model, gold = h.model, C.load(name.lower() + "_tiny.npz")
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    model.eval()
    with torch.no_grad():
        if name == "MGCN":
            fu, fi = model.forward(model.norm_adj)                   # no autograd: the gate / fuse / stacked-table route (a5b)
        elif name == "LayerGCN":
            model.forward_adj = model.norm_adj_matrix
            fu, fi = model.forward()
        else:
            fu, fi = model.forward()
    fwd_rel = max(G.rel_to(fu.numpy(), gold["fwd_u"]), G.rel_to(fi.numpy(), gold["fwd_i"]))
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
    score_err = float(np.abs(C.predict(model, gold) - gold["scores"]).max() / np.abs(gold["scores"]).max())
    out = {"model": name, "init_identical": bool(init_identical), "fwd_rel": fwd_rel, "loss": float(loss.item()),
           "want_loss": float(np.asarray(gold["loss"]).sum()), "grad_ok": bool(grad_ok), "score_err": score_err}
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_traj(key):
    """Two epochs of the training loop (`Trainer._train_epoch`, its Adam, its scheduler, its dataloader's shuffling and
    negative sampling) driving OUR class, against the trajectory the reference's class produced
    (tests/golden/traj_*_tiny.npz: every batch, every batch loss, per-epoch metrics)."""
    # key -> (model class, overrides of make_golden.py's dump_trajectory call, golden file)
    name, over, gfile = {"LightGCN": ("LightGCN", {"n_layers": [2], "reg_weight": [1e-4]}, "traj_lightgcn_tiny.npz"),
                         "FREEDOM": ("FREEDOM", {"dropout": [0.0], "reg_weight": [1e-3]}, "traj_freedom_tiny.npz"),
                         "FREEDOM-prune": ("FREEDOM", {"dropout": [0.8], "reg_weight": [1e-3]}, "traj_freedom_prune_tiny.npz"),
                         "LayerGCN": ("LayerGCN", {"dropout": [0.1]}, "traj_layergcn_tiny.npz"),
                         "BM3": ("BM3", {}, "traj_bm3_tiny.npz"),
                         "MGCN": ("MGCN", {}, "traj_mgcn_tiny.npz")}[key]
    h = C.build(name, over=over, after={"epochs": 2})
    gold = np.load(os.path.join(os.environ.get("MMREC_TRAJ_DIR", C.GOLDEN), gfile), allow_pickle=True)
    batches, losses = [], []
    orig = h.model.calculate_loss

    def spy(interaction):
        batches.append(interaction.numpy().copy())
        l = orig(interaction)
        losses.append(float(sum(l)) if isinstance(l, tuple) else float(l))
        return l
    h.model.calculate_loss = spy
    # The reference's own loader reproduces its shuffling and negative-sampling stream, so its batches are compared.  The
    # package's loader keeps the reference's batch format but draws its own stream (vectorised sampling), so with the
    # package harness the recorded batches are replayed and every loss and metric is compared.
    replay = not os.environ.get("MMREC_REFERENCE_SRC")
    # LayerGCN's uniform pruning draws from Python's `random`, the stream the reference's loader samples negatives from:
    # its state at the start of each epoch is recorded from the reference run (MMREC_RECORD_DIR) and restored in replay.
    state_file = os.path.join(C.GOLDEN, "traj_%s_tiny_pyrandom.npz" % key.lower())
    states = []

    def before_epoch(ep):
        if replay and os.path.isfile(state_file):
            st = np.load(state_file)["state%d" % ep]
            random.setstate((int(st[0]), tuple(int(x) for x in st[1:-1]), None))
        states.append(np.array([random.getstate()[0]] + list(random.getstate()[1]) + [0], dtype=np.int64))
    out = C.replay_trajectory(h, gold, before_epoch, epochs=None if replay else [h.train_data] * 2)
    if not replay and os.environ.get("MMREC_RECORD_DIR"):
        np.savez(os.path.join(os.environ["MMREC_RECORD_DIR"], "traj_%s_tiny_pyrandom.npz" % key.lower()),
                 **{"state%d" % ep: st for ep, st in enumerate(states)})
    batches = np.concatenate(batches, axis=1)
    out.update({"model": name, "batches": "recorded, replayed" if replay else "drawn by the reference's loader",
                "same_batches": bool(batches.shape == gold["batches"].shape and np.array_equal(batches, gold["batches"])),
                "first_loss": losses[0], "last_loss": losses[-1], "want_last_loss": float(gold["losses"][-1])})
    C.emit(out)


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    if arg.startswith("traj:"):
        main_traj(arg[5:])
    else:
        main_mmgcn() if arg == "mmgcn" else (main_model(arg) if arg else main())
