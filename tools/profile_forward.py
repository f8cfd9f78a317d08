"""Kernel-by-kernel device time of one inference `forward` at bench.py's shape (torch.profiler, eager launches, no CUDA graph).
    python tools/profile_forward.py [--workload baby] [--iters 10] [--out DIR]
Builds the model exactly as bench.py does (model class through the dataset on disk), flushes the L2 before every forward
and prints, per kernel of the forward, its median device time and the median gap since the previous kernel ended, then the
span first-start -> last-end.  With --out, the table is also written as DIR/profile_forward_<model>_<workload>.json."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="baby", choices=["baby", "sports", "clothing", "small", "tiny"])
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--out", default=None)
a = ap.parse_args()

dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
model_name = bench.MODEL_OF[a.workload]
wl = bench.Workload(a.workload, n_layers=3 if model_name == "FREEDOM" else 2)
_, _, _, model = bench.build_model(wl, model_name, dev, {"n_ui_layers": wl.n_layers} if model_name == "FREEDOM" else None)
model.eval()
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)

with torch.no_grad():
    for _ in range(3):                                              # lazy inits: occupancy queries, workspaces
        bench.forward_eval(model)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(a.iters):
            flush.zero_()
            torch.cuda.synchronize()
            with torch.profiler.record_function("forward"):
                bench.forward_eval(model)
            torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))["traceEvents"]

# device work of each `forward`: the kernels / memsets / copies whose launch (runtime call, linked by correlation id) falls
# inside that forward's record_function range on the host
spans = sorted((e["ts"], e["ts"] + e["dur"]) for e in trace if e.get("ph") == "X" and e.get("name") == "forward"
               and e.get("cat") == "user_annotation")
launch_ts = {e["args"]["correlation"]: e["ts"] for e in trace
             if e.get("ph") == "X" and e.get("cat") == "cuda_runtime" and "correlation" in e.get("args", {})}
dev_ev = [e for e in trace if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")
          and "correlation" in e.get("args", {})]
per_iter = [[] for _ in spans]
for e in dev_ev:
    t = launch_ts.get(e["args"]["correlation"])
    if t is None:
        continue
    for i, (t0, t1) in enumerate(spans):
        if t0 <= t <= t1:
            per_iter[i].append(e)
            break
per_iter = [sorted(k, key=lambda e: e["ts"]) for k in per_iter if k]
n_k = len(per_iter[0])
if any(len(k) != n_k for k in per_iter):
    raise SystemExit(f"the forwards launched different kernel sequences: {[len(k) for k in per_iter]}")

rows = []
for j in range(n_k):
    durs = [k[j]["dur"] for k in per_iter]
    gaps = [k[j]["ts"] - (k[j - 1]["ts"] + k[j - 1]["dur"]) for k in per_iter] if j else [0.0] * len(per_iter)
    rows.append({"name": per_iter[0][j]["name"], "grid": per_iter[0][j]["args"].get("grid"),
                 "us": float(np.median(durs)), "gap_before_us": float(np.median(gaps))})
span = float(np.median([k[-1]["ts"] + k[-1]["dur"] - k[0]["ts"] for k in per_iter]))
props = torch.cuda.get_device_properties(dev)
try:
    import subprocess
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except Exception:                                                   # noqa: BLE001
    power = "unknown"
print(f"{model_name} / {a.workload}: forward(norm_adj) under no_grad, eager, L2 flushed; median of {len(per_iter)} forwards "
      f"on {props.name} (power limit {power})")
for r in rows:
    print(f"  {r['us']:8.2f} us  gap {r['gap_before_us']:6.2f} us  grid {r['grid']}  {r['name'][:110]}")
print(f"  kernels {sum(r['us'] for r in rows):.2f} us, gaps {sum(r['gap_before_us'] for r in rows):.2f} us, span {span:.2f} us")
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, f"profile_forward_{model_name}_{a.workload}.json"), "w") as f:
        json.dump({"model": model_name, "workload": a.workload, "device": props.name, "power_limit": power,
                   "forwards": len(per_iter), "kernels": rows, "span_us": span}, f, indent=1)
