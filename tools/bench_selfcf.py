"""SELFCFED_LGN measurement: one training step (`calculate_loss` + backward + `FusedAdam.step`) at the baby, sports and
clothing shapes (synthetic graphs of those sizes, d = 64, n_layers = 1 and 2, B = 2048), with the encoder's per-batch edge
dropout taken three ways:
  (a) "mask":    the keep bits of the draw (`ops.edge_keep_bits`) and K1 with the edge-keep mask on the fixed CSR and plan,
                 forward and backward (`ops.propagate_mean_dropped`) -- what the model runs;
  (b) "rebuild": the kept entries rebuilt with `CSR.from_coo` (sort, new plan, host syncs) every step, and the backward's
                 `CSR.t()` built from it, through `ops.propagate_mean`;
  (c) "torch":   the reference's expression on the device (`sparse_dropout` builds a sparse COO tensor of the kept entries,
                 then `torch.sparse.mm` per layer, stack and mean; encoders.py:77-112).
The rest of the step (predictor, target dropouts, cosine losses, L2 term) is the same torch code for all three.  The host
draw (`np.random.random()`, `torch.rand(nnz)` on the CPU, copied to the device) is the same for all three routes and is timed
apart; the timed steps take draws made before the timed window, so they measure the device work of the step.  The three
routes' losses on the same draws are compared (relative difference).

Device events after a warm-up, `--reps` repetitions per route, the routes interleaved step by step (median and range).  The card name, power limit and maximum SM clock are
read (read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lgmrec import card, timed  # noqa: E402


class Setup:
    def __init__(self, shape, n_layers, B, seed=0):
        from mmrec_b200 import graph
        from mmrec_b200.utils import synth
        u, i, e, d, _ = synth.SHAPES[shape]
        g = synth.make_graph(u, i, e, seed=seed).split(0)
        self.nu, self.ni, self.L, self.B = u, i, n_layers, B
        ur, ic = g[0], g[1]
        self.A = graph.build_norm_adj((ur, ic), u, i, "cuda")
        draw_of, mirror = graph.dropout_entry_maps(ur, ic, u, i)
        self.draw_of, self.mirror = torch.from_numpy(draw_of).cuda(), torch.from_numpy(mirror).cuda()
        r, c, v = self.A.coo()
        perm = torch.empty_like(self.draw_of)
        perm[self.draw_of.long()] = torch.arange(self.A.nnz, device="cuda", dtype=perm.dtype)
        p = perm.long()
        self.ref_adj = torch.sparse_coo_tensor(torch.stack((r[p], c[p])), v[p], (u + i, u + i))   # the reference's stored order
        self.coo = (r, c, v)
        torch.manual_seed(seed)
        self.user_emb = torch.nn.Parameter(torch.nn.init.xavier_uniform_(torch.empty(u, d, device="cuda")))
        self.item_emb = torch.nn.Parameter(torch.nn.init.xavier_uniform_(torch.empty(i, d, device="cuda")))
        self.predictor = torch.nn.Linear(d, d).cuda()
        from mmrec_b200.optim import FusedAdam
        self.opt = FusedAdam([self.user_emb, self.item_emb] + list(self.predictor.parameters()), lr=1e-3)
        gen = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.users = torch.randint(0, u, (B,), device="cuda", generator=gen)
        self.items = torch.randint(0, i, (B,), device="cuda", generator=gen)

    def draw(self):
        rate = np.random.random()
        return rate, torch.rand(self.A.nnz).to("cuda")

    def propagate(self, route, ego, rate, draws):
        from mmrec_b200 import ops
        from mmrec_b200.ops import CSR
        kp, scale = float(np.float32(1 - rate)), float(np.float32(1. / (1 - rate)))
        if route == "mask":
            keep, keep_t = ops.edge_keep_bits(draws, kp, self.draw_of, self.mirror)
            return ops.propagate_mean_dropped(self.A, ego, self.L, keep, keep_t, scale)
        if route == "rebuild":
            r, c, v = self.coo
            k = torch.floor(draws[self.draw_of.long()] + kp) != 0
            C = CSR.from_coo(r[k], c[k], v[k] * scale, self.A.n_rows, self.A.n_cols, sum_duplicates=False, symmetric=False)
            return ops.propagate_mean(C, ego, self.L)
        x = self.ref_adj                                              # encoders.py:77-88, 99-104
        random_tensor = 1 - rate
        random_tensor += draws
        mask = torch.floor(random_tensor).type(torch.bool)
        a = torch.sparse_coo_tensor(x._indices()[:, mask], x._values()[mask], x.shape) * (1. / (1 - rate))
        layers = [ego]
        for _ in range(self.L):
            ego = torch.sparse.mm(a, ego)
            layers.append(ego)
        return torch.stack(layers, dim=1).mean(dim=1)

    def step(self, route, draw=None):
        rate, draws = self.draw() if draw is None else draw
        ego = torch.cat([self.user_emb, self.item_emb], 0)
        all_e = self.propagate(route, ego, rate, draws)
        u_on, i_on = all_e[:self.nu][self.users], all_e[self.nu:][self.items]
        with torch.no_grad():
            u_t, i_t = F.dropout(u_on.clone(), 0.1), F.dropout(i_on.clone(), 0.1)
        reg = (u_on ** 2).sum() * 0.5 + (i_on ** 2).sum() * 0.5
        pu, pi = self.predictor(u_on), self.predictor(i_on)
        loss = -F.cosine_similarity(pu, i_t, dim=-1).mean() / 2 - F.cosine_similarity(pi, u_t, dim=-1).mean() / 2 + 0.1 * reg
        loss.backward()
        self.opt.step()
        self.opt.zero_grad()
        return loss.detach()


def run_shape(shape, n_layers, B, reps):
    s = Setup(shape, n_layers, B)
    res = {"shape": shape, "n_layers": n_layers, "B": B, "n_nodes": s.A.n_rows, "nnz": s.A.nnz}
    # the same draw through the three routes, from the same weights: the losses must agree to fp32 reorder error
    np.random.seed(1)
    torch.manual_seed(1)
    draw = s.draw()
    state = [p.detach().clone() for p in (s.user_emb, s.item_emb, s.predictor.weight, s.predictor.bias)]
    losses = {}
    for route in ("mask", "rebuild", "torch"):
        with torch.no_grad():
            for p, q in zip((s.user_emb, s.item_emb, s.predictor.weight, s.predictor.bias), state):
                p.copy_(q)
        torch.manual_seed(2)
        torch.cuda.manual_seed(2)
        losses[route] = float(s.step(route, draw))
    res["loss"] = losses
    res["loss_rel_diff_vs_torch"] = {k: abs(v - losses["torch"]) / abs(losses["torch"]) for k, v in losses.items()}
    for _ in range(3):
        s.draw()
    res["host_draw_and_copy"] = timed(s.draw, reps)
    routes = ("mask", "rebuild", "torch")
    for route in routes:
        for _ in range(3):
            s.step(route)                                             # warm-up
    draws = [s.draw() for _ in range(reps)]
    ts = {r: [] for r in routes}
    for k in range(reps):                                             # interleaved: drift and neighbours hit every route alike
        for route in routes:
            ts[route].append(timed(lambda: s.step(route, draws[k]), 1)["median_s"])
    for route in routes:
        t = sorted(ts[route])
        res[route] = {"median_s": t[len(t) // 2], "min_s": t[0], "max_s": t[-1]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60)
    ap.add_argument("--shapes", default="baby,sports,clothing")
    ap.add_argument("--layers", default="1,2")
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"card": card(), "runs": [run_shape(sh, int(L), a.batch, a.reps) for sh in a.shapes.split(",") for L in a.layers.split(",")]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
