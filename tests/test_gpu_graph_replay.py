"""What bench.py times is replayed from CUDA graphs: the sections here are checked in that form, against eager calls.

Every timed section of bench.py ([A] the inference propagation, [B] the projections, [C] / [C4096] `full_sort_topk`, and the
end-to-end forms with pinned host copies inside the graph) is captured once on a side stream and replayed, with the
embedding tables rewritten in place between replays.  The eager tests pin eager calls only.  Here:

1. Every drop-in model's sections, captured after two warm-up calls, replay bit for bit like a fresh eager call: twice in a
   row (self-cleaning counters, state carried from one replay to the next), and after the inputs were rewritten in place
   (tables through `.data`, the captured `users` / `mask` buffers refilled with a shuffled mask, columns outside the
   catalogue and a user without mask entries).  The top-k after the rewrite is also checked against an fp64 re-score of the
   same fp32 embeddings (near-tie rule), so a replay equal to a wrong eager call fails too.  Each check runs on device
   buffers and in the end-to-end form (pinned host -> device copies, the section, device -> host copies, one graph).
2. Ops on one CSR with split rows and CTA tasks, launched with different operands on two streams at once, each equal to its
   serial result; and a graph replay on one stream beside eager calls on another.
3. Entry points that read a count back to the host refuse to be captured before they enqueue anything; the capture is
   abandoned cleanly and the same stream then runs them eagerly.
4. The peer exchange and barrier (world size 1) replayed from a graph: the call counter in `state[0]` advances once per
   call, so nothing about the barrier is baked into the graph.
"""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu

SEED = 1234
TOPK = 50
EVAL_BATCH = 128                                # tiny has 300 users: batches of 128, 128 and a ragged 44


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    from mmrec_b200.utils import synth
    _lib.require_device()
    tmp = tempfile.mkdtemp(prefix="mmrec_gpu_")
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(os.path.join(tmp, "data"), "tiny", g, v, t)
    return os.path.join(tmp, "data") + "/"


def build(model_name, data_path, overrides):
    from mmrec_b200.utils.configurator import Config
    from mmrec_b200.utils.dataloader import TrainDataLoader
    from mmrec_b200.utils.dataset import RecDataset
    from mmrec_b200.utils.utils import get_model, init_seed
    cfg = {"data_path": data_path, "eval_batch_size": 128, "train_batch_size": 512}
    cfg.update(overrides)
    config = Config(model_name, "tiny", cfg)
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    tr, _, _ = RecDataset(config).split()
    train = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    init_seed(config["seed"])
    train.pretrain_setup()
    model = get_model(model_name)(config, train).to(config["device"])
    return config, train, model


def _section_a_default(model):
    model.invalidate_eval_cache()
    return model._score_embeddings()


def _section_a_stored(model):
    model.forward()                              # stores the table full_sort_* scores (MMGCN `result`, MVGAE `result_embed`)
    return model._score_embeddings()


# name -> (golden file with the reference's initial parameters or None, config overrides, section A, tensors besides the
# parameters that the sections read and a caller may rewrite, scores ranked through a sigmoid)
MODELS = {
    "BM3": ("bm3_tiny.npz", {}, _section_a_default, (), False),
    "FREEDOM": ("freedom_tiny.npz", {"n_ui_layers": 3}, _section_a_default, (), False),
    "LayerGCN": ("layergcn_tiny.npz", {}, _section_a_default, (), False),
    "LightGCN": ("lightgcn_tiny.npz", {"n_layers": [3]}, _section_a_default, (), False),
    "LGMRec": (None, {}, _section_a_default, (), False),
    "MGCN": ("mgcn_tiny.npz", {}, _section_a_default, (), False),
    "MMGCN": (None, {}, _section_a_stored, ("id_embedding", "result"), False),
    "MVGAE": (None, {}, _section_a_stored, ("result_embed",), False),
    "SELFCFED_LGN": (None, {}, _section_a_default, (), False),
    "SLMRec": (None, {}, lambda m: m.compute(), ("all_users", "all_items"), True),
}


def _flat(out):
    if torch.is_tensor(out):
        return [out]
    return [t for o in out for t in _flat(o)] if isinstance(out, (tuple, list)) else []


def _assert_equal(got, want, what):
    got, want = _flat(got), _flat(want)
    assert len(got) == len(want) and got, what
    for j, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and torch.equal(g.to(w.device), w), f"{what}: output {j} differs"


def _tables(model, extra):
    """What a caller may rewrite in place: every floating-point parameter and the model's stored tables."""
    ts = [p for p in model.parameters() if p.is_floating_point()]
    ts += [getattr(model, a) for a in extra if getattr(model, a, None) is not None]
    assert ts
    return ts


def _new_values(t, step):
    """Other values of the same magnitude (a row-reversed mix), deterministic per step."""
    x = t.detach()
    if x.dim() == 0:
        return x * 0.5
    return (x.flip(0) * (0.5 + 0.125 * step) + x * 0.375).contiguous()


def _capture(fn, side):
    """Two warm-up calls on the side stream, then one capture there (bench.py's order)."""
    with torch.cuda.stream(side), torch.no_grad():
        for _ in range(2):
            torch.cuda.manual_seed(SEED)
            fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g, stream=side):
        out = fn()
    torch.cuda.synchronize()
    return g, out


def _replay(g, side):
    torch.cuda.manual_seed(SEED)                 # LGMRec draws in every forward: the replay and the eager call share the draws
    with torch.cuda.stream(side):
        g.replay()
    torch.cuda.synchronize()


def _eager(fn):
    torch.cuda.manual_seed(SEED)
    with torch.no_grad():
        out = fn()
    torch.cuda.synchronize()
    return [t.clone() for t in _flat(out)]


def _train_mask(train, lo, hi):
    coo = train.inter_matrix(form="coo")
    r, c = np.asarray(coo.row, dtype=np.int64), np.asarray(coo.col, dtype=np.int64)
    m = (r >= lo) & (r < hi)
    o = np.lexsort((c[m], r[m]))
    return np.stack([r[m][o] - lo, c[m][o]])


def _new_batch(rng, B, nnz, n_users, n_items):
    """New contents of the same shapes: other users, and a mask in no particular order (the unsorted route), with columns
    outside [0, n_items) and batch row 0 without entries."""
    users = rng.permutation(n_users)[:B].astype(np.int64)
    rows = rng.integers(1, B, nnz) if B > 1 else np.zeros(nnz, dtype=np.int64)
    cols = rng.integers(0, n_items, nnz)
    out = rng.random(nnz) < 0.1
    cols[out] = rng.choice(np.array([-7, -1, n_items, n_items + 5]), int(out.sum()))
    mask = np.stack([rows, cols]).astype(np.int64)
    assert (np.diff(rows) < 0).any() and out.any()
    if B > 1:
        assert not (rows == 0).any()
    return users, mask


def _check_topk_fp64(idx, u, i, users, mask, sigmoid):
    """The top-k against an fp64 re-score of the same fp32 embeddings: every index that differs from the exact ranking
    (ties to the lower index) must be a near tie (test_gpu_configs.near_tie_check's rule)."""
    s = u.detach().cpu().double()[torch.from_numpy(users)] @ i.detach().cpu().double().t()
    if sigmoid:
        s = torch.sigmoid(s)
    keep = (mask[1] >= 0) & (mask[1] < s.shape[1]) & (mask[0] >= 0) & (mask[0] < s.shape[0])
    s[mask[0][keep], mask[1][keep]] = -1e10
    _, ri = O.topk_tie_low_index(s.numpy(), idx.shape[1])
    scale = float(s[s > -1e9].abs().max())
    got = idx.cpu().numpy()
    for b in np.nonzero((got != ri).any(axis=1))[0]:
        cols = np.nonzero(got[b] != ri[b])[0]
        gap = np.abs(s[b, got[b, cols]].numpy() - s[b, ri[b, cols]].numpy()).max()
        assert gap < 4e-6 * scale, f"row {b}: top-k differs from the fp64 re-score beyond a near tie (gap {gap})"


_PINNED = []      # pinned buffers a captured copy reads or writes: kept for the whole run, as bench.py keeps its own


class _Section:
    """One section on device buffers or in the end-to-end form.  `inputs`: device tensors the section reads (rewritten in
    place on update); in the e2e form each has a pinned host twin copied in inside the graph, and the outputs are copied
    out to pinned host buffers inside the graph."""

    def __init__(self, fn, inputs, e2e, dev):
        self.fn, self.inputs, self.e2e = fn, inputs, e2e
        if not e2e:
            self.run = fn
            return
        self.host_in = [t.detach().cpu().pin_memory() for t in inputs]
        with torch.no_grad():
            torch.cuda.manual_seed(SEED)
            shapes = [t for t in _flat(fn())]
        self.host_out = [torch.empty(t.shape, dtype=t.dtype).pin_memory() for t in shapes]
        _PINNED.extend(self.host_in + self.host_out)

        def run():
            for t, h in zip(self.inputs, self.host_in):
                t.data.copy_(h, non_blocking=True)
            out = _flat(fn())
            for h, t in zip(self.host_out, out):
                h.copy_(t, non_blocking=True)
            return self.host_out
        self.run = run

    def set_inputs(self, values):
        torch.cuda.synchronize()
        if self.e2e:
            for h, v in zip(self.host_in, values):
                h.copy_(v)
        for t, v in zip(self.inputs, values):    # (the e2e graph copies them in itself; the eager reference reads these)
            t.data.copy_(v)
        torch.cuda.synchronize()


def _check_section(what, sec, side, new_values, after=None):
    """(a) two replays == a fresh eager call; (b) after `new_values` are written in place, the replay == the eager call.
    `after(eager_outputs)`: the further check (c) on the eager result after the rewrite."""
    g, out = _capture(sec.run, side)
    for rep in ("first", "second"):
        for t in _flat(out):                     # a replay that skips work leaves this behind
            t.fill_(-3)
        _replay(g, side)
        got = [t.clone() for t in _flat(out)]
        _assert_equal(got, _eager(sec.fn), f"{what}: {rep} replay")
    sec.set_inputs(new_values)
    _replay(g, side)
    got = [t.clone() for t in _flat(out)]
    want = _eager(sec.fn)
    _assert_equal(got, want, f"{what}: replay after the inputs were rewritten in place")
    if after is not None:
        after(want)
    return g


@pytest.mark.parametrize("form", ["device", "e2e"])
@pytest.mark.parametrize("name", list(MODELS))
def test_model_sections_replay_equal_eager(env, golden, monkeypatch, name, form):
    """[C] (all users, and batches with a ragged last one), [A] and, for FREEDOM, [B], replayed from graphs as bench.py
    replays them, equal to eager calls before and after the inputs change in place; [C] also against fp64.  The graphs are
    planned with 64 non-zeros per task and CTA tasks from 17 on, so that the tiny graphs have split rows (items of degree
    66 .. 152) and CTA tasks, as the graphs of real datasets have at the default plan."""
    from mmrec_b200 import ops
    gold, over, sec_a, extra, sigmoid = MODELS[name]
    monkeypatch.setattr(ops, "SEG", 64)
    monkeypatch.setattr(ops, "LIGHT_MAX", 16)
    config, train, model = build(name, env, over)
    csrs = [v for m in model.modules() for v in vars(m).values() if isinstance(v, ops.CSR)]
    assert any(A.n_split > 0 and A.n_cta_tasks > 0 for A in csrs), "no graph with split rows and CTA tasks"
    dev = config["device"]
    if gold is not None:
        g = golden(gold)
        model.load_state_dict({k[7:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param0.")}, strict=True)
    model.eval()
    e2e = form == "e2e"
    rng = np.random.default_rng(sum(map(ord, name + form)))
    side = torch.cuda.Stream()
    with torch.no_grad():
        torch.cuda.manual_seed(SEED)
        if name == "SLMRec":                     # SLMRec scores the tables its last training step stored
            model.all_users, model.all_items = model.compute()
        elif sec_a is _section_a_stored:
            model.forward()
    torch.cuda.synchronize()
    n_users, n_items = model.n_users, model.n_items
    tables = _tables(model, extra)
    step = [0]

    def rewritten_tables():
        step[0] += 1
        return [_new_values(t, step[0]) for t in tables]

    def embeddings():
        torch.cuda.manual_seed(SEED)
        with torch.no_grad():
            return model._stored_tables() if name == "SLMRec" else model._score_embeddings()

    # ---- [C]: full_sort_topk with the evaluation cache warm (captured first: [A] drops the cache) ----
    spans = [(0, n_users)] + [(lo, min(n_users, lo + EVAL_BATCH)) for lo in range(0, n_users, EVAL_BATCH)]
    assert spans[-1][1] - spans[-1][0] < EVAL_BATCH
    for lo, hi in spans:
        users = torch.arange(lo, hi, device=dev)
        mask = torch.from_numpy(_train_mask(train, lo, hi)).to(dev)
        sec = _Section(lambda: model.full_sort_topk([users, mask], TOPK), [users, mask] + tables, e2e, dev)
        nu, nm = _new_batch(rng, hi - lo, mask.shape[1], n_users, n_items)
        new = [torch.from_numpy(nu).to(dev), torch.from_numpy(nm).to(dev)] + rewritten_tables()

        def fp64(want, nu=nu, nm=nm):
            u, i = embeddings()
            _check_topk_fp64(want[0], u, i, nu, nm, sigmoid)
        _check_section(f"{name} [C] users {lo}..{hi} ({form})", sec, side, new, fp64)
    # ---- [A]: the inference propagation behind full_sort_* ----
    saved = {a: getattr(model, a) for a in extra}
    sec = _Section(lambda: sec_a(model), tables, e2e, dev)
    _check_section(f"{name} [A] ({form})", sec, side, rewritten_tables())
    for a, t in saved.items():                   # (the capture left graph-pool tensors in the stored attributes)
        setattr(model, a, t)
    model.invalidate_eval_cache()
    # ---- [B]: FREEDOM's two projections over the whole feature tables ----
    if name == "FREEDOM":
        def sec_b():
            return (ops.project(model.image_embedding.weight, model.image_trs.weight, model.image_trs.bias),
                    ops.project(model.text_embedding.weight, model.text_trs.weight, model.text_trs.bias))
        sec = _Section(sec_b, tables, e2e, dev)
        _check_section(f"{name} [B] ({form})", sec, side, rewritten_tables())


@pytest.mark.parametrize("k", [TOPK, 1])
def test_score_topk_replay_after_tables_rewritten(env, k):
    """The fused scoring with the item operand packed inside the call (no `Catalog`: the route of the models that do not
    cache their embeddings, and of `max_dot` at k = 1), at a catalogue large enough for the fused kernels at k = 50 (the
    tiny models' 120 items are not).  Replays equal eager calls, and after both tables, the users and the mask were
    rewritten in place, equal the exact ranking of the new integer scores."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(17 + k)
    n_users, I, d, B = 900, 2000, 64, 700
    ints = lambda shape: torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, shape, 2, density=0.5), 1.0)).cuda()
    U, T = ints((n_users, d)), ints((I, d))
    users = torch.arange(B, device="cuda")
    mask = torch.from_numpy(np.stack([np.repeat(np.arange(B), 4), rng.integers(0, I, 4 * B)])).cuda()
    sec = _Section(lambda: ops.score_topk(U, T, users, mask, k), [U, T, users, mask], False, "cuda")
    nu, nm = _new_batch(rng, B, mask.shape[1], n_users, I)
    new = [ints((n_users, d)), ints((I, d)), torch.from_numpy(nu).cuda(), torch.from_numpy(nm).cuda()]

    def exact(want):
        s = U.cpu().double()[torch.from_numpy(nu)] @ T.cpu().double().t()
        keep = (nm[1] >= 0) & (nm[1] < I)
        s[nm[0][keep], nm[1][keep]] = -1e10
        wv, wi = O.topk_tie_low_index(s.numpy(), k)
        assert np.array_equal(want[1].cpu().numpy(), wi) and np.array_equal(want[0].cpu().double().numpy(), wv)
    _check_section(f"score_topk k={k}", sec, torch.cuda.Stream(), new, exact)


def test_itemknncbf_scoring_is_refused_under_capture(env):
    """ItemKNNCBF has no propagation ([A]): its scores come straight from the interaction CSR and the item kNN graph.  Its
    [C], `sparse_score_topk` (K9), reads back how many rows need the unfused route, so it cannot be captured: the capture is
    refused before anything is enqueued, and the same stream then scores eagerly, bit-identical to the unfused route.  (A
    device-side exact route for K9 would make it capturable; that is a kernel of its own, not part of these tests.)"""
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    config, train, model = build("ItemKNNCBF", env, {})
    dev = config["device"]
    model.eval()
    users = torch.arange(0, model.n_users, device=dev)
    mask = torch.from_numpy(_train_mask(train, 0, model.n_users)).to(dev)
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with pytest.raises(MMRecError, match="sparse_score_topk reads a result back"):
            with torch.no_grad(), torch.cuda.graph(g, stream=side):
                model.full_sort_topk([users, mask], TOPK)
        assert not torch.cuda.is_current_stream_capturing()
        with torch.no_grad():
            idx = model.full_sort_topk([users, mask], TOPK)
            _, want = ops.mask_topk(ops.sparse_scores(model.r_matrix, model.item_sim, users), mask, TOPK)
    torch.cuda.synchronize()
    assert torch.equal(idx, want)


# ======================================================================================================================
# 2. one CSR on two streams at once
# ======================================================================================================================
ROW_LENS = [0, 0, 1, 7, 32, 33, 64, 511, 512, 513, 520, 4200, 0, 3]   # test_gpu_exact_arith: split rows 513, 520, 4200
N = 4500                                                                # square, so that propagate_mean runs on it
COPIES = 6                                                              # launches enqueued back to back per stream


@pytest.fixture(scope="module")
def sq(env):
    """A square CSR with the split rows (513, 520, 4200 non-zeros) and CTA tasks of test_gpu_exact_arith, |v| <= 3 in units of
    1/8, plus its transpose."""
    from mmrec_b200.ops import CSR
    rng = np.random.default_rng(5)
    lens = ROW_LENS + list(rng.integers(0, 24, N - len(ROW_LENS)))
    row = np.concatenate([np.full(n, r, dtype=np.int64) for r, n in enumerate(lens)])
    col = np.concatenate([np.sort(rng.choice(N, size=n, replace=False)).astype(np.int64) for n in lens])
    vals = O.exact_ints(rng, row.shape, 2)
    vals[vals == 0] = 1
    dev = torch.device("cuda:0")
    A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev),
                     torch.from_numpy(O.to_f32_exact(vals, 2.0 ** -3)).to(dev), N, N)
    assert A.n_split == 3 and A.n_cta_tasks >= 1 and A.longest_row == 4200
    A.t()                                                               # built now: the backward must not build it mid-flight
    import scipy.sparse as sp
    return A, sp.csr_matrix((vals, (row, col)), shape=(N, N))


def _gate(streams):
    """Hold both streams behind one spin kernel so that everything enqueued after this starts together (overlap is more
    likely; correctness does not depend on it)."""
    torch.cuda.synchronize()
    torch.cuda._sleep(20_000_000)
    ev = torch.cuda.Event()
    ev.record()
    for s in streams:
        s.wait_event(ev)


def _two_streams(op, operands):
    """op(operand) -> tensors; run serially on one stream, then COPIES times per stream on two streams, interleaved, with no
    synchronisation between the launches.  Returns (serial, [per stream: [per copy: outputs]])."""
    serial = [[t.clone() for t in _flat(op(x))] for x in operands]
    torch.cuda.synchronize()
    s = [torch.cuda.Stream(), torch.cuda.Stream()]
    _gate(s)
    outs = [[], []]
    for _ in range(COPIES):
        for k in (0, 1):
            with torch.cuda.stream(s[k]):
                outs[k].append(_flat(op(operands[k])))
    torch.cuda.synchronize()
    return serial, outs, s


def _assert_streams(serial, outs, what):
    for k in (0, 1):
        for c, o in enumerate(outs[k]):
            _assert_equal(o, serial[k], f"{what}: stream {k}, copy {c}")


def _counters_zero(A, streams):
    for s in list(streams) + [torch.cuda.current_stream()]:
        with torch.cuda.stream(s):
            assert int(A.counters.abs().sum().item()) == 0


@pytest.mark.parametrize("d", [32, 64, 96, 128, 192, 256])
def test_spmm_two_streams(sq, d):
    """spmm_raw at every vector width with different X per stream: each stream's Y is the exact product, and every stream's
    split-row counters are back to zero."""
    from mmrec_b200 import ops
    A, Ai = sq
    rng = np.random.default_rng(d)
    Xi = [O.exact_ints(rng, (N, d), 1) for _ in range(2)]
    X = [torch.from_numpy(O.to_f32_exact(x, 0.5)).cuda() for x in Xi]

    def op(x):
        y = torch.empty(N, d, device=x.device)
        ops.spmm_raw(A, x, Y=y)
        return y
    serial, outs, s = _two_streams(op, X)
    for k in (0, 1):
        O.assert_bits(serial[k][0], O.to_f32_exact(Ai @ Xi[k], 2.0 ** -4), f"d={d} serial {k}")
    _assert_streams(serial, outs, f"spmm d={d}")
    _counters_zero(A, s)


def test_spmm_drop_two_streams(sq):
    """The edge-dropout kernel (`mmrec_spmm_drop_f32`) with different keep bits and X per stream."""
    from mmrec_b200 import ops
    A, Ai = sq
    rng = np.random.default_rng(11)
    d = 64
    X = [torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (N, d), 1), 0.5)).cuda() for _ in range(2)]
    words = (A.nnz + 31) // 32
    keep = [torch.from_numpy(rng.integers(-2 ** 31, 2 ** 31, words).astype(np.int32)).cuda() for _ in range(2)]

    def op(k):
        y = torch.empty(N, d, device="cuda")
        ops.spmm_raw(A, X[k], Y=y, drop=(keep[k], 2.0))
        return y
    serial, outs, s = _two_streams(op, [0, 1])
    assert not torch.equal(serial[0][0], serial[1][0])
    _assert_streams(serial, outs, "spmm drop")
    _counters_zero(A, s)


def test_propagate_mean_two_streams(sq):
    """propagate_mean forward and backward (on the transpose) with different E_0 and upstream gradients per stream."""
    from mmrec_b200 import ops
    A, _ = sq
    rng = np.random.default_rng(12)
    d = 64
    E = [torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (N, d), 1), 0.5)).cuda() for _ in range(2)]
    G = [torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (N, d), 2), 0.25)).cuda() for _ in range(2)]

    def op(k):
        e = E[k].clone().requires_grad_(True)
        out = ops.propagate_mean(A, e, 2)
        gx, = torch.autograd.grad(out, e, G[k])
        return out.detach(), gx
    serial, outs, s = _two_streams(op, [0, 1])
    _assert_streams(serial, outs, "propagate_mean")
    _counters_zero(A, s)
    _counters_zero(A.t(), s)


def test_score_topk_and_max_dot_two_streams(env):
    """score_topk (the item operand packed inside the call, in each stream's workspace) and max_dot with different
    operands per stream; integer scores, so every correct ranking is one bit pattern."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(13)
    B, I, d = 700, 2000, 64
    U = [torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (B, d), 2, density=0.5), 1.0)).cuda() for _ in range(2)]
    T = [torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (I, d), 2, density=0.5), 1.0)).cuda() for _ in range(2)]
    serial, outs, _ = _two_streams(lambda k: ops.score_topk(U[k], T[k], None, None, TOPK), [0, 1])
    for k in (0, 1):
        s = U[k].cpu().double() @ T[k].cpu().double().t()
        wv, wi = O.topk_tie_low_index(s.numpy(), TOPK)
        assert np.array_equal(serial[k][1].cpu().numpy(), wi) and np.array_equal(serial[k][0].cpu().double().numpy(), wv)
    _assert_streams(serial, outs, "score_topk")
    with torch.no_grad():
        serial, outs, _ = _two_streams(lambda k: ops.max_dot(U[k], T[k]), [0, 1])
    _assert_streams(serial, outs, "max_dot")


def test_graph_replay_beside_eager_on_another_stream(sq):
    """A captured SpMM replayed on one stream while the same CSR runs eagerly with other operands on a second stream."""
    from mmrec_b200 import ops
    A, Ai = sq
    rng = np.random.default_rng(14)
    d = 64
    Xi = [O.exact_ints(rng, (N, d), 1) for _ in range(2)]
    X = [torch.from_numpy(O.to_f32_exact(x, 0.5)).cuda() for x in Xi]
    want = [torch.from_numpy(O.to_f32_exact(Ai @ x, 2.0 ** -4)).cuda() for x in Xi]
    s = [torch.cuda.Stream(), torch.cuda.Stream()]
    Yg = torch.empty(N, d, device="cuda")
    g, _ = _capture(lambda: ops.spmm_raw(A, X[0], Y=Yg), s[0])
    _gate(s)
    Ye = []
    for _ in range(COPIES):
        with torch.cuda.stream(s[0]):
            g.replay()
        with torch.cuda.stream(s[1]):
            Ye.append(torch.empty(N, d, device="cuda"))
            ops.spmm_raw(A, X[1], Y=Ye[-1])
    torch.cuda.synchronize()
    assert torch.equal(Yg, want[0])
    for c, y in enumerate(Ye):
        assert torch.equal(y, want[1]), f"eager copy {c}"
    _counters_zero(A, s)


# ======================================================================================================================
# 3. entry points that read back refuse to be captured
# ======================================================================================================================
def _refused(what, call, check):
    """`call` inside a capture raises MMRecError naming `what`; the capture ends cleanly and the same stream then runs
    `call` eagerly, checked by `check(result)`."""
    from mmrec_b200._lib import MMRecError
    side = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with pytest.raises(MMRecError, match=f"{what} reads a result back"):
            with torch.no_grad(), torch.cuda.graph(g, stream=side):
                call()
        assert not torch.cuda.is_current_stream_capturing()
        out = call()
    torch.cuda.synchronize()
    check(out)


def test_readback_entry_points_refuse_capture(sq):
    """knn_topk, sparse_score_topk, CSR.from_coo / the plan, and the fallback diagnostics: refused under capture; then
    eager on the same stream with the right bits.  (sparse_scores never reads back: it is capturable.)"""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    A, Ai = sq
    rng = np.random.default_rng(15)
    n, F, k = 600, 256, 10
    x = torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (n, F), 1, density=0.2), 1.0)).cuda()
    sim = x.cpu().double() @ x.cpu().double().t()
    _, wi = O.topk_tie_low_index(sim.numpy(), k)
    _refused("knn_topk", lambda: ops.knn_topk(x, k), lambda o: np.testing.assert_array_equal(o[1].cpu().numpy(), wi))
    r, c, v = A.coo()
    _refused("CSR.from_coo", lambda: CSR.from_coo(r, c, v, N, N),
             lambda B: (torch.equal(B.rowptr, A.rowptr) and torch.equal(B.colidx, A.colidx) and torch.equal(B.vals, A.vals))
             or pytest.fail("CSR rebuilt eagerly differs"))
    _refused("CSR._plan", lambda: CSR(N, N, A.rowptr, A.colidx, A.vals, A.nnz),
             lambda B: (B.n_split == A.n_split and torch.equal(B.tasks, A.tasks)) or pytest.fail("plan differs"))
    R = CSR.from_coo(*(t for t in A.coo()[:2]), torch.ones(A.nnz, device="cuda"), N, N)
    users = torch.arange(0, 300, device="cuda")
    mask = torch.stack([torch.arange(300, device="cuda"), torch.arange(300, device="cuda") * 7 % N])
    want = ops.mask_topk(ops.sparse_scores(R, A, users), mask, k)[1]
    _refused("sparse_score_topk", lambda: ops.sparse_score_topk(R, A, users, mask, k),
             lambda o: torch.equal(o[1], want) or pytest.fail("sparse_score_topk differs from the unfused route"))
    for name in ("fused_fallback_rows", "knn_fallback_rows", "sparse_topk_fallback_rows"):
        _refused(name, getattr(ops, name), lambda v: isinstance(v, int) or pytest.fail(name))


# ======================================================================================================================
# 4. the peer exchange and barrier replayed from a graph (world size 1)
# ======================================================================================================================
def test_peer_exchange_and_barrier_replay_advance_the_call_counter(env):
    """World size 1: the barriers wait on the flags this rank wrote itself.  `peer_exchange` (final layer: (acc + part) /
    div) and `peer_barrier` captured together and replayed N times: the output equals `peer_reduce_push` and the float64
    sum bit for bit; `state[0]` (the call number) advances by one per call, and the block counter `state[2]` is back to 0."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(16)
    n, div, reps = 4096 * 4, 4.0, 5
    part = torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (n,), 12), 2.0 ** -6)).cuda()
    acc = torch.from_numpy(O.to_f32_exact(O.exact_ints(rng, (n,), 12), 2.0 ** -6)).cuda()
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    state = torch.zeros(4, dtype=torch.int32, device="cuda")
    dst = torch.empty(n, device="cuda")
    want64 = (acc.cpu().double() + part.cpu().double()) / div
    ref = torch.empty(n, device="cuda")
    ops.peer_reduce_push([part.data_ptr()], [ref.data_ptr()], n, 0, acc_in=acc, acc_div=div, final_layer=True)

    def fn():
        ops.peer_exchange([part.data_ptr()], [dst.data_ptr()], [flags.data_ptr()], state, n, 0, acc_in=acc, acc_div=div,
                          final_layer=True)
        ops.peer_barrier([flags.data_ptr()], state, 0)
    side = torch.cuda.Stream()
    g, _ = _capture(fn, side)
    s0 = int(state[0].item())
    assert s0 == 4 and int(state[2].item()) == 0  # the two warm-up rounds, two calls each
    for r in range(reps):
        dst.fill_(-1.0)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dst, ref) and torch.equal(dst.cpu().double(), want64), f"replay {r}"
        st = state.cpu().tolist()
        assert st[0] == s0 + 2 * (r + 1) and st[2] == 0, f"replay {r}: state {st}"
