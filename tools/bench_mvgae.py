"""MVGAE measurement.  (1) `ops.max_dot` forward + backward (K3's fused score + top-1, then a gather and `index_sum_rows`)
against the reference's expression under autograd (`torch.max(torch.sum(z[users.repeat(1, B)] * z[neg_items], -1), -1)`,
mvgae.py:76-84: a [B, B, d] tensor) at B in {1024, 2048, 4096}, d = 64, M = B; torch is capped at 4096, where each such
tensor is 4 GiB.  Time, peak memory above the inputs (after a warm-up, so K3's cached workspace is not counted: its size is
reported beside), and whether the two argmax agree.  (2) One MVGAE training step (`calculate_loss` + backward +
`FusedAdam.step`) at the baby shape with B = 2048, the same step with the decode replaced by the reference's expression, and
one full `Trainer.evaluate`.

Device events after a warm-up, `--reps` repetitions (median and range).  The card name, power limit and maximum SM clock are
read (read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lgmrec import card, timed  # noqa: E402


def ref_decode(z, user, neg_items):
    """mvgae.py:76-84 without the sigmoid."""
    re_users = torch.unsqueeze(user, 1).repeat(1, neg_items.size(0))
    return torch.max(torch.sum(z[re_users] * z[neg_items], -1), dim=-1)


def op_vs_torch(B, d, reps, torch_cap):
    from mmrec_b200 import _lib, ops
    g = torch.Generator(device="cuda").manual_seed(B)
    N = 2 * B
    z0 = torch.sigmoid(torch.randn(N, d, generator=g, device="cuda"))
    user = torch.randint(0, N, (B,), generator=g, device="cuda")
    neg = torch.randint(0, N, (B,), generator=g, device="cuda")
    w = torch.randn(B, generator=g, device="cuda")
    res = {"B": B, "M": B, "d": d, "k3_workspace_mib": _lib.load().mmrec_score_topk_workspace_bytes(B, B, d, 1) / 2 ** 20}
    outs = {}

    def run(kind):
        z = z0.clone().requires_grad_(True)
        v, i = ops.max_dot(z[user], z[neg]) if kind == "max_dot" else ref_decode(z, user, neg)
        (w * v).sum().backward()
        outs[kind] = (v.detach(), i, z.grad)

    for kind in ("max_dot", "torch"):
        if kind == "torch" and B > torch_cap:
            res[kind] = {"skipped": f"B > {torch_cap}: {B * B * d * 4 / 2 ** 30:.0f} GiB per [B, B, d] tensor"}
            continue
        try:
            run(kind)                                                  # warm-up
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            run(kind)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            res[kind] = dict(timed(lambda: run(kind), reps), peak_mib=peak / 2 ** 20)
        except torch.cuda.OutOfMemoryError as e:
            res[kind] = {"error": "out of memory: " + str(e).splitlines()[0]}
        outs.pop("torch", None) if kind == "torch" and "error" in res[kind] else None
        torch.cuda.empty_cache()
    if "max_dot" in outs and "torch" in outs:
        a, b = outs["max_dot"], outs["torch"]
        res["argmax_differs"] = int((a[1] != b[1]).sum())
        res["max_rel_diff"] = {"values": float(((a[0] - b[0]).abs().max() / b[0].abs().max()).item()),
                               "dz": float(((a[2] - b[2]).abs().max() / b[2].abs().max()).item())}
        if "median_s" in res["max_dot"] and "median_s" in res["torch"]:
            res["speedup"] = res["torch"]["median_s"] / res["max_dot"]["median_s"]
    return res


def train_step(shape, reps, batch_size):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.utils import synth
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_mvgae_")
    u, i, e, d, f = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), shape, gr, v, t)
    config = Config("MVGAE", shape, {"data_path": os.path.join(tmp, "data") + "/", "train_batch_size": batch_size})
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("MVGAE")(config, train).to(config["device"])
    trainer = Trainer(config, model)
    batch = next(iter(train)).to(config["device"])
    model.train()

    def step():
        trainer.optimizer.zero_grad()
        model.calculate_loss(batch).backward()
        trainer.optimizer.step()
    step()
    res = {"shape": shape, "users": u, "items": i, "edges": e, "F": f, "batch": int(batch.shape[1]),
           "optimizer": type(trainer.optimizer).__name__}
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    res["step"] = timed(step, reps)
    res["step"]["peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    # the same step with the four decodes taken by the reference's [B, B, d] expression
    real = ops.max_dot
    # (q = z[user], t = z[neg_items]: q[rows.repeat(1, M)] is the reference's gathered [B, M, d] operand z[re_users])
    ops.max_dot = lambda q, t: torch.max(torch.sum(
        q[torch.arange(q.shape[0], device=q.device)[:, None].repeat(1, t.shape[0])] * t, -1), dim=-1)
    try:
        step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        res["step_torch_decode"] = timed(step, reps)
        res["step_torch_decode"]["peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    except torch.cuda.OutOfMemoryError as e:
        res["step_torch_decode"] = {"error": "out of memory: " + str(e).splitlines()[0]}
    finally:
        ops.max_dot = real
        torch.cuda.empty_cache()
    # the four decodes of the step alone, on the step's shapes (z over all nodes, B users and negatives)
    N, B = u + i, int(batch.shape[1])
    z = torch.sigmoid(torch.randn(N, config["embedding_size"], device="cuda"))

    def decodes():
        for _ in range(4):
            zz = z.clone().requires_grad_(True)
            ops.max_dot(zz[batch[0]], zz[batch[2]])[0].sum().backward()
    decodes()
    res["decodes"] = timed(decodes, reps)
    res["decode_share"] = res["decodes"]["median_s"] / res["step"]["median_s"]
    model.eval()
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(1, reps // 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="1024,2048,4096,8192")
    ap.add_argument("--torch-cap", type=int, default=4096)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"card": card(), "op": [op_vs_torch(int(b), 64, a.reps, a.torch_cap) for b in a.sizes.split(",")]}
    if not a.skip_train:
        out["train"] = [train_step("baby", a.reps, 2048)]
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
