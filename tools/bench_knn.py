"""K7 measurement: the kNN build of one modality (F = 4096, k = 10 by default) -- `ops.knn_topk` (tensor-core certified
filter, csrc/knn_cf.cu) against the route it replaces (`ops.score` on the exact CUDA-core kernel + `ops.mask_topk` in row
blocks), at the item counts of baby (7 000), clothing (23 000), one GPU's share of configs[4] (125 037) and 10^6.

Device events around each call, after a warm-up of both routes; the new route repeated `--reps` times, the old one
`--old-reps` times up to `--old-max` items, outputs compared bitwise at every size where both ran.  The approximate pass's
tensor rate comes from its kernel time in a separate torch.profiler run (2 m_pad n_pad F_pad flops of wgmma f16).  The card
name and power limit are read in the same run.  Prints the result as JSON (and writes it to --out if given)."""
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
    except Exception as e:                                            # (the number is still the device's; say where the card info failed)
        q = f"nvidia-smi unavailable: {e}"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def table(n, F, seed):
    """N(0,1) rows, L2-normalised as graph._knn does, built in slices (the 10^6 x 4096 table is 16 GB)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(n, F, device="cuda")
    for s in range(0, n, 65536):
        blk = torch.randn(min(65536, n - s), F, generator=g, device="cuda")
        x[s:s + blk.shape[0]] = blk.div(torch.norm(blk, p=2, dim=-1, keepdim=True))
    return x


def old_route(cn, k):
    from mmrec_b200 import ops
    step = max(128, (256 << 20) // (4 * cn.shape[0]))
    vals, inds = [], []
    for s in range(0, cn.shape[0], step):
        v, i = ops.mask_topk(ops.score(cn[s:s + step], cn), None, k)
        vals.append(v); inds.append(i)
    return torch.cat(vals), torch.cat(inds)


def timed(fn, reps):
    out, ts = None, []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return out, ts


def pass_kernel_seconds(cn, k):
    from torch.profiler import ProfilerActivity, profile
    from mmrec_b200 import ops
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.knn_topk(cn, k)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = "pass" if "knn_pass_kernel" in e.name else ("final" if "knn_final_kernel" in e.name else
                                                               ("thr" if "knn_thr_kernel" in e.name else ("pack" if "knn_pack" in e.name else None)))
            if name:
                per[name] = per.get(name, 0.0) + e.device_time_total / 1e6
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="7000,23000,125037,1000000")
    ap.add_argument("--F", type=int, default=4096)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--old-reps", type=int, default=2)
    ap.add_argument("--old-max", type=int, default=125037)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn: needs a CUDA device")
    from mmrec_b200 import ops
    res = {"card": card(), "F": a.F, "k": a.k, "rows": []}
    w = table(3000, a.F, 0)                                           # warm-up: modules, attributes, both routes
    ops.knn_topk(w, a.k); old_route(w, a.k)
    del w
    for n in [int(s) for s in a.sizes.split(",")]:
        cn = table(n, a.F, n)
        new, t_new = timed(lambda: ops.knn_topk(cn, a.k), a.reps if n < 500000 else max(1, a.reps - 1))
        row = {"n": n, "new_s": t_new, "fallback_rows": ops.knn_fallback_rows()}
        per = pass_kernel_seconds(cn, a.k)
        m_pad = (n + 255) // 256 * 256
        n_pad = (n + 127) // 128 * 128
        kp = (a.F + 63) // 64 * 64
        flops = 2.0 * m_pad * n_pad * kp
        row["kernel_s"] = per
        if per.get("pass"):
            row["pass_tflops"] = flops / per["pass"] / 1e12
            row["pass_share_of_989"] = row["pass_tflops"] / 989.0
        if n <= a.old_max:
            old, t_old = timed(lambda: old_route(cn, a.k), a.old_reps)
            row["old_s"] = t_old
            row["speedup_median"] = sorted(t_old)[len(t_old) // 2] / sorted(t_new)[len(t_new) // 2]
            row["bitwise_equal"] = bool(torch.equal(new[0].view(torch.int32), old[0].view(torch.int32)) and torch.equal(new[1], old[1]))
            del old
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
        del cn, new
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
