"""ItemKNNCBF measurement: model initialisation and full evaluation, the new route (K7's shrink route -> kNN CSR, K9 sparse
scores / fused sparse top-k) against the reference's torch route on the same device (`torch.norm`, `mm` -> `div` -> `topk`
-> scatter into a dense [I, I] -> `torch.sparse.mm(R, item_sim)` into a dense [U, I] kept for evaluation; evaluation =
row gather, mask, `torch.topk`).

Shapes: the synthetic graphs of mmrec_b200.utils.synth for baby, sports and clothing with F = 8192 concatenated feature
columns (two modalities of 4096), knn_k = 10, shrink = 10, top-50 over every user in batches of 4096 with the train
positives masked.  At 125 037 items (`xls`) only the new route runs; the torch route's memory is computed from shapes.
Device events around each phase (after one warm-up of each route at the first shape), peak memory from
torch.cuda.max_memory_allocated above the feature table.  The card name and power limit are read in the same run.
Prints JSON (and writes it to --out if given)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:
        q = f"nvidia-smi unavailable: {e}"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3


def batch_mask(R, users):
    """The trainer's mask for a batch: (batch row, item) of every train positive, from the interaction CSR."""
    start, end = R.rowptr[users].long(), R.rowptr[users + 1].long()
    cnt = end - start
    rows = torch.repeat_interleave(torch.arange(users.numel(), device=users.device), cnt)
    off = torch.arange(int(cnt.sum()), device=users.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    return torch.stack([rows, R.colidx[torch.repeat_interleave(start, cnt) + off].long()])


def new_init(X, R_coo, n_users, n_items, k, shrink):
    from mmrec_b200 import ops
    r, c, v = R_coo
    R = ops.CSR.from_coo(r, c, v, n_users, n_items)
    val, idx = ops.knn_topk(X, k, norms=torch.norm(X, p=2, dim=-1), shrink=shrink)
    S = ops.CSR.from_coo(torch.arange(n_items, device=X.device).repeat_interleave(k), idx.reshape(-1), val.reshape(-1), n_items, n_items)
    return R, S


def torch_init(X, R_coo, n_users, n_items, k, shrink):
    r, c, v = R_coo
    R = torch.sparse_coo_tensor(torch.stack([r, c]), v, (n_users, n_items))
    i_norm = torch.norm(X, p=2, dim=-1, keepdim=True)
    sim = torch.mm(X, X.T).div(i_norm * i_norm.T + shrink)
    knn_val, knn_ind = torch.topk(sim, k, dim=-1)
    item_sim = torch.zeros_like(sim).scatter_(-1, knn_ind, knn_val)
    del sim
    return torch.sparse.mm(R, item_sim)


def evaluate(R, users_all, k, topk_fn):
    out = []
    for s in range(0, users_all.numel(), 4096):
        u = users_all[s:s + 4096]
        out.append(topk_fn(u, batch_mask(R, u)))
    return out


def run_shape(name, F, k, shrink, torch_route, seed=0):
    from mmrec_b200 import ops
    from mmrec_b200.utils import synth
    U, I, E, _, _ = synth.SHAPES[name]
    if name == "xls":
        I = 125037                                                    # one GPU's share of configs[4]'s items
    g = synth.make_graph(U, I, E, seed=seed)
    tr_u, tr_i = g.train
    dev = torch.device("cuda:0")
    R_coo = (torch.as_tensor(tr_u, dtype=torch.int64, device=dev), torch.as_tensor(tr_i, dtype=torch.int64, device=dev),
             torch.ones(len(tr_u), dtype=torch.float32, device=dev))
    X = torch.randn(I, F, generator=torch.Generator(device="cuda").manual_seed(seed + 1), device=dev)
    res = {"users": U, "items": I, "train_edges": int(len(tr_u)), "F": F}
    users_all = torch.arange(U, device=dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    (R, S), res["new_init_s"] = timed(lambda: new_init(X, R_coo, U, I, k, shrink))
    res["new_init_fallback_rows"] = ops.knn_fallback_rows()
    _, res["new_eval_fused_s"] = timed(lambda: evaluate(R, users_all, 50, lambda u, m: ops.sparse_score_topk(R, S, u, m, 50)))
    res["new_eval_fused_fallback_rows_last_batch"] = ops.sparse_topk_fallback_rows()
    _, res["new_eval_unfused_s"] = timed(lambda: evaluate(R, users_all, 50, lambda u, m: ops.mask_topk(ops.sparse_scores(R, S, u), m, 50)))
    res["new_peak_gib_above_table"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    res["torch_route_dense_bytes_from_shapes"] = 4 * I * I * 4 + 4 * U * I
    if torch_route:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        sm, res["torch_init_s"] = timed(lambda: torch_init(X, R_coo, U, I, k, shrink))

        def tk(u, m):
            s = sm[u]
            s[m[0], m[1]] = -1e10
            return torch.topk(s, 50, dim=-1)
        _, res["torch_eval_s"] = timed(lambda: evaluate(R, users_all, 50, tk))
        res["torch_peak_gib_above_table"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        del sm
    else:
        res["torch_init_s"] = res["torch_eval_s"] = res["torch_peak_gib_above_table"] = "not measured"
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="baby,sports,clothing,xls")
    ap.add_argument("--F", type=int, default=8192)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--shrink", type=float, default=10.0)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from mmrec_b200 import _lib
    _lib.require_device()
    result = {"card": card(), "F": a.F, "knn_k": a.k, "shrink": a.shrink, "shapes": {}}
    run_shape("tiny", 256, a.k, a.shrink, True)                       # warm-up of both routes
    for name in a.shapes.split(","):
        result["shapes"][name] = run_shape(name, a.F, a.k, a.shrink, torch_route=(name != "xls"))
        print(name, json.dumps(result["shapes"][name]), flush=True)
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
