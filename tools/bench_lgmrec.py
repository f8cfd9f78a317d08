"""LGMRec measurement.  (1) K8, `ops.expsum_rows` forward + backward, against torch's expression under autograd
(`torch.exp(torch.matmul(q, t.T) / tau).sum(dim=1)`, lgmrec.py:164) at B = 2048 and M in {7 050, 19 445, 36 000, 40 000,
250 000}, d = 64: time, peak memory above the inputs, the output difference and the share of the 3xTF32 tensor rate.
(2) One LGMRec training step (`calculate_loss` + backward + `FusedAdam.step`) at the baby shape (H = 4) and the clothing
shape (H = 64, two hypergraph layers), the time of the contrastive sums inside it, and one full `Trainer.evaluate`.

Device events after a warm-up, `--reps` repetitions (median and range).  The card name, power limit and maximum SM clock are
read (read-only) in the same run.  Prints JSON; writes it to --out only when given."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

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


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    ts.sort()
    return {"median_s": ts[len(ts) // 2], "min_s": ts[0], "max_s": ts[-1]}


def kernel_vs_torch(B, M, d, reps, tf32x3_peak):
    from mmrec_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    q0 = torch.nn.functional.normalize(torch.randn(B, d, generator=g, device="cuda"))
    t0 = torch.nn.functional.normalize(torch.randn(M, d, generator=g, device="cuda"))
    up = torch.rand(B, generator=g, device="cuda")
    res = {"B": B, "M": M, "d": d}
    outs = {}

    def run(kind):
        q, t = q0.clone().requires_grad_(True), t0.clone().requires_grad_(True)
        if kind == "k8":
            ttl = ops.expsum_rows(q, t, 0.2)
        else:
            ttl = torch.exp(torch.matmul(q, t.T) / 0.2).sum(dim=1)
        ttl.backward(up)
        outs[kind] = (ttl.detach(), q.grad, t.grad)

    for kind in ("k8", "torch"):
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
        torch.cuda.empty_cache()
    if "median_s" in res["k8"]:
        # five [B, M, d] contractions of 2 B M d flops: the forward's, and per backward output the recomputed scores + the
        # weighted sum; each is three tf32 passes, so the rate is compared with a third of the TF32 peak
        flops = 2 * B * M * d * 5
        res["k8"]["tf32x3_share"] = flops / res["k8"]["median_s"] / tf32x3_peak
    if "k8" in outs and "torch" in outs:
        res["max_rel_diff"] = {n: float(((a - b).abs().max() / b.abs().max()).item())
                               for n, a, b in zip(("ttl", "dq", "dt"), outs["k8"], outs["torch"])}
    return res


def train_step(shape, over, reps):
    from mmrec_b200 import ops
    from mmrec_b200.common.trainer import Trainer
    from mmrec_b200.utils import synth
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import EvalDataLoader, TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    tmp = tempfile.mkdtemp(prefix="mmrec_bench_lgmrec_")
    u, i, e, d, f = synth.SHAPES[shape]
    gr = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), shape, gr, v, t)
    config = Config("LGMRec", shape, dict({"data_path": os.path.join(tmp, "data") + "/"}, **over))
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    ds = RecDataset(config)
    tr, va, te = ds.split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model("LGMRec")(config, train).to(config["device"])
    trainer = Trainer(config, model)
    batch = next(iter(train)).to(config["device"])
    model.train()

    def step():
        trainer.optimizer.zero_grad()
        model.calculate_loss(batch).backward()
        trainer.optimizer.step()
    step()
    res = {"shape": shape, "users": u, "items": i, "edges": e, "F": f, "hyper_num": config["hyper_num"],
           "n_hyper_layer": config["n_hyper_layer"], "batch": int(batch.shape[1]), "step": timed(step, reps)}
    # the contrastive sums of the step: K8 forward + backward on the step's shapes (users and items, B = batch)
    B = int(batch.shape[1])
    qs = [torch.randn(B, d, device="cuda") for _ in range(2)]
    ts = [torch.randn(n, d, device="cuda") for n in (u, i)]

    def sums():
        for q, t_ in zip(qs, ts):
            qq, tt = q.clone().requires_grad_(True), t_.clone().requires_grad_(True)
            ops.expsum_rows(qq, tt, 0.2).sum().backward()
    sums()
    res["contrastive_sums"] = timed(sums, reps)
    res["contrastive_share"] = res["contrastive_sums"]["median_s"] / res["step"]["median_s"]
    model.eval()
    res["evaluate"] = timed(lambda: trainer.evaluate(valid), max(1, reps // 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="7050,19445,36000,40000,250000")
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--tf32x3-peak", type=float, default=494e12 / 3,
                    help="tensor rate of 3xTF32 in flop/s (default: the H100 SXM data-sheet dense TF32 figure / 3)")
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = {"card": card(), "kernel": [kernel_vs_torch(2048, int(m), 64, a.reps, a.tf32x3_peak) for m in a.sizes.split(",")]}
    if not a.skip_train:
        out["train"] = [train_step("baby", {}, a.reps),
                        train_step("clothing", {"n_hyper_layer": [2], "hyper_num": [64], "keep_rate": [0.2], "alpha": [0.2]}, a.reps)]
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
