"""Is `cpu_baseline.kind = "port"` a faithful stand-in for the reference's own speed?  Needs an unmodified enoche/MMRec
checkout (MMREC_REFERENCE_SRC=<checkout>/src): runs the UNMODIFIED reference FREEDOM (`src/models/freedom.py`, via tests/golden/ref_loader.py) and the
oracle port (`oracle/mmrec_oracle.py`, what `bench.py --impl reference` times) on the same baby-shaped synthetic dataset, same
thread count, and prints the time of `forward` and of one `full_sort_predict` + mask + top-50 batch for both.
    python tools/ref_vs_port_timing.py [--threads 8]
"""
import argparse, json, os, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
ap = argparse.ArgumentParser(); ap.add_argument("--threads", type=int, default=os.cpu_count()); ap.add_argument("--reps", type=int, default=5)
a = ap.parse_args()
torch.set_num_threads(a.threads)
import ref_loader
from mmrec_b200.utils import synth
from oracle import mmrec_oracle as O
ref_loader.install()
tmp = tempfile.mkdtemp(prefix="mmrec_refcmp_")
data = ref_loader.run_dir(tmp)
U, I, E, d, F = synth.SHAPES["baby"]
g = synth.make_graph(U, I, E, seed=0)
v, t = synth.make_features(I, F, seed=1)
synth.write_dataset(data, "baby", g, v, t)
import logging; logging.disable(logging.CRITICAL)
from utils.configurator import Config
from utils.dataset import RecDataset
from utils.dataloader import TrainDataLoader, EvalDataLoader
from utils.utils import init_seed, get_model
config = Config("FREEDOM", "baby", {"gpu_id": 0, "use_gpu": False, "n_ui_layers": 3})
config["inter_file_name"] = "baby.inter"
config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
for k in config["hyper_parameters"]:
    if isinstance(config[k], list):
        config[k] = config[k][0]
ds = RecDataset(config); str(ds)
tr, va, te = ds.split(); str(tr), str(va), str(te)
train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
valid = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
init_seed(config["seed"]); train.pretrain_setup()
t0 = time.perf_counter()
model = get_model("FREEDOM")(config, train)
t_init = time.perf_counter() - t0
model.eval()
eb = next(iter(valid))


def med(fn):
    ts = []
    for _ in range(a.reps + 1):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return float(np.median(ts[1:]))


with torch.no_grad():
    ref_fwd = med(lambda: model.forward(model.norm_adj))

    def ref_eval():
        s = model.full_sort_predict(eb)
        s[eb[1][0], eb[1][1]] = -1e10
        torch.topk(s, 50, dim=-1)
    ref_ev = med(ref_eval)
    # the port, on the reference's own matrices and parameters
    adj, mm = model.norm_adj, model.mm_adj
    ue, ie = model.user_embedding.weight.detach(), model.item_id_embedding.weight.detach()
    port_fwd = med(lambda: O.freedom_forward(adj, mm, ue, ie, int(config["n_mm_layers"]), int(config["n_ui_layers"])))
    u_g, i_g = O.freedom_forward(adj, mm, ue, ie, int(config["n_mm_layers"]), int(config["n_ui_layers"]))
    ru, ri = model.forward(model.norm_adj)
    same = bool(torch.equal(u_g, ru) and torch.equal(i_g, ri))

    def port_eval():
        s = O.full_sort_scores(u_g, i_g, eb[0])
        O.mask_topk(s, eb[1], 50)
    port_ev = med(port_eval)
print(json.dumps({"threads": a.threads, "users": U, "items": I, "edges": int(len(g.train[0])), "eval_batch": int(eb[0].numel()),
                  "reference_init_s": round(t_init, 2), "reference_forward_ms": round(ref_fwd * 1e3, 2), "port_forward_ms": round(port_fwd * 1e3, 2),
                  "reference_eval_batch_ms": round(ref_ev * 1e3, 2), "port_eval_batch_ms": round(port_ev * 1e3, 2),
                  "forward_outputs_bit_identical": same}))
