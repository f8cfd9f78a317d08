"""Host-side operators over the C ABI (include/mmrec_b200.h): the three op families of MMRec's hot path.

Each function here replaces a PyTorch library call of the reference (cited per function, paths relative
to the root of enoche/MMRec) with a call into libmmrec_b200.so on the current CUDA stream.  PyTorch is used for
device memory, streams and autograd bookkeeping only.  There is no CPU path: tensors must live on a
sm_90 device, otherwise `MMRecError` is raised.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import MMRecError, check

_ws_cache: dict = {}
import os as _os
SEG = int(_os.environ.get("MMREC_SPMM_SEG", "512"))        # non-zeros per SpMM task (rows longer than this are split)
LIGHT_MAX = int(_os.environ.get("MMREC_SPMM_LIGHT", "32"))  # tasks longer than this are run by a whole CTA


def launch_count() -> int:
    """Kernels of this library launched by this process so far: every launch site in the C ABI counts itself
    (`mmrec_launch_count`); bench.py's `gpu_launches` is the difference over its timed region (for a section replayed
    from a CUDA graph: the launches recorded while capturing it, times the replays)."""
    return int(_lib.load().mmrec_launch_count())


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise MMRecError("mmrec_b200 ops run on CUDA tensors only (no CPU fallback)")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise MMRecError(f"expected float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _refuse_capture(op: str):
    """Raise before anything is enqueued when the current stream is capturing a CUDA graph: `op` reads a count back to the
    host (a synchronising copy), which would invalidate the capture, or bake the count seen at capture time into the graph."""
    if torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing():     # (no capture before CUDA is set up)
        raise MMRecError(f"{op} reads a result back to the host and cannot be captured in a CUDA graph: run it eagerly")


def _ws(name: str, nbytes: int, device) -> torch.Tensor:
    """Scratch for one op family, per device AND per stream (two streams never share a buffer).  A buffer that turned
    out too small is kept alive next to its replacement: a CUDA graph captured earlier has its address baked in."""
    key = (name, device.index, torch.cuda.current_stream(device).cuda_stream)
    bufs = _ws_cache.setdefault(key, [])
    if not bufs or bufs[-1].numel() < nbytes:
        grow = int(bufs[-1].numel() * 1.5) if bufs else 0
        bufs.append(torch.empty(max(int(nbytes), grow, 256), dtype=torch.uint8, device=device))
    return bufs[-1]


# ------------------------------------------------------------------------------------------------
# K1c: CSR container
# ------------------------------------------------------------------------------------------------
class CSR:
    """Row-sorted int32 CSR of a sparse matrix on the device, with the SpMM work plan.

    Stands in for the reference's `torch.sparse` COO tensors (`norm_adj`, `masked_adj`, `mm_adj`, `R`;
    SURVEY.md 8a a1/a2/a8).  Built once per graph (per epoch for FREEDOM's pruned graph) instead of the
    coalesce + COO->CSR conversion ATen performs inside every `torch.sparse.mm` call.
    """

    def __init__(self, n_rows, n_cols, rowptr, colidx, vals, nnz, symmetric=False, seg=None, light_max=None):
        self.n_rows, self.n_cols, self.nnz = int(n_rows), int(n_cols), int(nnz)
        self.rowptr, self.colidx, self.vals = rowptr, colidx, vals
        self.symmetric = symmetric
        self.seg = SEG if seg is None else seg
        self.light_max = LIGHT_MAX if light_max is None else light_max
        self._t: Optional["CSR"] = None
        self._split = {}                                # (device, stream) -> split-row counters and partials, see _split_scratch
        self._plan()

    # -- construction ------------------------------------------------------------------------------
    @staticmethod
    def from_coo(row: torch.Tensor, col: torch.Tensor, val: Optional[torch.Tensor], n_rows: int, n_cols: int,
                 sum_duplicates: bool = True, symmetric: bool = False, seg=None, light_max=None) -> "CSR":
        _refuse_capture("CSR.from_coo")
        _lib.require_device()
        _need_cuda(row, col, val)
        lib = _lib.load()
        row, col = row.to(torch.int64).contiguous(), col.to(torch.int64).contiguous()
        val = None if val is None else _f32c(val)
        nnz = row.numel()
        dev = row.device
        rowptr = torch.empty(n_rows + 1, dtype=torch.int32, device=dev)
        colidx = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        vals = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
        nnz_out = torch.zeros(1, dtype=torch.int64, device=dev)
        nbytes = lib.mmrec_csr_from_coo_workspace_bytes(nnz, n_rows)
        ws = _ws("csr", nbytes, dev)
        check(lib.mmrec_csr_from_coo(nnz, _ptr(row), _ptr(col), _ptr(val), n_rows, n_cols, int(sum_duplicates),
                                     _ptr(rowptr), _ptr(colidx), _ptr(vals), _ptr(nnz_out), _ptr(ws), ws.numel(),
                                     _stream()), "mmrec_csr_from_coo")
        n = int(nnz_out.item())
        return CSR(n_rows, n_cols, rowptr, colidx[:max(n, 1)], vals[:max(n, 1)], n, symmetric, seg, light_max)

    @staticmethod
    def from_torch_sparse(t: torch.Tensor, symmetric: bool = False) -> "CSR":
        """From an (un-coalesced) torch COO tensor as the reference builds them."""
        idx, val = t._indices(), t._values()
        return CSR.from_coo(idx[0], idx[1], val.to(torch.float32), t.shape[0], t.shape[1], True, symmetric)

    def _plan(self):
        _refuse_capture("CSR._plan")
        lib = _lib.load()
        dev = self.rowptr.device
        max_tasks = self.n_rows + self.nnz // self.seg + 1
        max_split = self.nnz // self.seg + 1
        tasks = torch.empty(4 * max_tasks, dtype=torch.int32, device=dev)
        split = torch.empty(4 * max_split, dtype=torch.int32, device=dev)
        counts = torch.zeros(8, dtype=torch.int64, device=dev)
        ws = _ws("plan", lib.mmrec_spmm_plan_workspace_bytes(self.n_rows, max_tasks), dev)
        check(lib.mmrec_spmm_plan(self.n_rows, _ptr(self.rowptr), self.seg, self.light_max, max_tasks, _ptr(tasks), _ptr(split),
                                  _ptr(counts), _ptr(ws), ws.numel(), _stream()), "mmrec_spmm_plan")
        c = counts.tolist()
        self.n_tasks, self.n_split, self.n_slots, self.longest_row = int(c[0]), int(c[1]), int(c[2]), int(c[3])
        self.n_cta_tasks = int(c[4])
        self.tasks = tasks[:4 * max(self.n_tasks, 1)]
        self.split_rows = split[:4 * max(self.n_split, 1)]

    def _split_scratch(self):
        """The split rows' arrival counters and segment partials of the current stream, per device AND per stream like `_ws`:
        two products of this matrix in flight on two streams must not count each other's segments or add each other's
        partials.  The counters are zero at rest (the last segment of a row resets its counter).  Buffers are never dropped,
        so a CUDA graph that captured their addresses stays valid.  Counters first allocated while the stream is capturing
        are zeroed by a memset inside that graph; they are zeroed again (in the graph being captured, or eagerly) until an
        eager call has done it."""
        dev = self.rowptr.device
        key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
        s = self._split.get(key)
        if s is None:
            s = self._split[key] = {"counters": torch.zeros(max(self.n_split, 1), dtype=torch.int32, device=dev), "partial": {},
                                    "zeroed": not torch.cuda.is_current_stream_capturing()}
        elif not s["zeroed"]:
            s["counters"].zero_()
            s["zeroed"] = not torch.cuda.is_current_stream_capturing()
        return s

    @property
    def counters(self) -> torch.Tensor:
        """The split-row arrival counters of the current stream (all zero between products)."""
        return self._split_scratch()["counters"]

    def partial(self, d: int) -> torch.Tensor:
        """The segment partials of the current stream for width d."""
        parts = self._split_scratch()["partial"]
        t = parts.get(d)
        if t is None:
            t = parts[d] = torch.empty(max(self.n_slots, 1) * d, dtype=torch.float32, device=self.rowptr.device)
        return t

    # -- views ---------------------------------------------------------------------------------------
    def coo(self):
        """(row int64, col int64, val) of the stored entries."""
        counts = (self.rowptr[1:] - self.rowptr[:-1]).to(torch.int64)
        row = torch.repeat_interleave(torch.arange(self.n_rows, device=self.rowptr.device), counts)
        return row, self.colidx[:self.nnz].to(torch.int64), self.vals[:self.nnz]

    def t(self) -> "CSR":
        """Transposed matrix (needed by the backward of directed graphs: mm_adj, R)."""
        if self.symmetric:
            return self
        if self._t is None:
            r, c, v = self.coo()
            self._t = CSR.from_coo(c, r, v, self.n_cols, self.n_rows, False, False, self.seg, self.light_max)
            self._t._t = self
        return self._t

    def to_dense(self) -> torch.Tensor:
        r, c, v = self.coo()
        out = torch.zeros(self.n_rows, self.n_cols, dtype=torch.float32, device=v.device)
        out.index_put_((r, c), v, accumulate=True)
        return out

    def algorithmic_bytes(self, d: int) -> int:
        """SURVEY.md 8(d): 4(n_rows+1) + 8 nnz + 4 n_cols d + 4 n_rows d."""
        return 4 * (self.n_rows + 1) + 8 * self.nnz + 4 * self.n_cols * d + 4 * self.n_rows * d


# ------------------------------------------------------------------------------------------------
# K1: SpMM
# ------------------------------------------------------------------------------------------------
class PanelCSR:
    """A sparse matrix cut into column panels (each an ordinary `CSR` over all rows and the panel's columns only) for graphs
    whose dense operand does not fit the L2 (BASELINE config 5: 2M x 128 fp32 user table = 1 GB).  `spmm_raw` multiplies
    the panels one after the other, accumulating in Y, so that the rows of X a panel gathers -- `panel_bytes` of them -- are
    L2-resident: every row of X comes from HBM once per product instead of once per non-zero.  Same interface as `CSR` as far
    as the propagation needs it (`n_rows`, `n_cols`, `nnz`, `t()`, `algorithmic_bytes`)."""

    def __init__(self, n_rows, n_cols, panels, bounds, symmetric=False):
        self.n_rows, self.n_cols, self.panels, self.bounds, self.symmetric = n_rows, n_cols, panels, bounds, symmetric
        self.nnz = sum(p.nnz for p in panels)
        self.n_tasks = min(p.n_tasks for p in panels) if panels else 0
        self._t = None

    @staticmethod
    def from_coo(row, col, val, n_rows, n_cols, d, panel_bytes=48 << 20, sum_duplicates=True, symmetric=False) -> "PanelCSR":
        cols_per_panel = max(1024, panel_bytes // (4 * d))
        n_panels = max(1, -(-n_cols // cols_per_panel))
        cols_per_panel = -(-n_cols // n_panels)
        panels, bounds = [], []
        for p in range(n_panels):
            lo, hi = p * cols_per_panel, min(n_cols, (p + 1) * cols_per_panel)
            m = (col >= lo) & (col < hi)
            panels.append(CSR.from_coo(row[m], col[m], None if val is None else val[m], n_rows, n_cols, sum_duplicates, False))
            bounds.append((lo, hi))
        out = PanelCSR(n_rows, n_cols, panels, bounds, symmetric)
        out._coo = (row, col, val, d, panel_bytes, sum_duplicates)
        return out

    def t(self):
        if self.symmetric:
            return self
        if self._t is None:
            row, col, val, d, pb, sd = self._coo
            self._t = PanelCSR.from_coo(col, row, val, self.n_cols, self.n_rows, d, pb, sd, False)
            self._t._t = self
        return self._t

    def algorithmic_bytes(self, d: int) -> int:
        return 4 * (self.n_rows + 1) + 8 * self.nnz + 4 * self.n_cols * d + 4 * self.n_rows * d


def spmm_raw(A, X: torch.Tensor, Y: Optional[torch.Tensor] = None, acc_in: Optional[torch.Tensor] = None,
             acc_out: Optional[torch.Tensor] = None, acc_div: float = 1.0, gate_ref: Optional[torch.Tensor] = None,
             use_plan: bool = True, y_accumulate: bool = False, drop: Optional[tuple] = None):
    """y = A X with the fused epilogue of include/mmrec_b200.h (no autograd).  Replaces `torch.sparse.mm`
    (`src/models/freedom.py:167,172`) plus the stack/mean (`:175-176`) and `+ h` (`:178`) that follow.
    `drop` = (keep_bits, scale): only the entries whose keep bit is set take part, weighted fl(v * scale)
    (the edge-keep mask of `mmrec_spmm_op`; SelfCF's `sparse_dropout`, `src/common/encoders.py:77-88`)."""
    if drop is not None and (isinstance(A, PanelCSR) or gate_ref is not None or y_accumulate):
        raise MMRecError("spmm: the edge-keep mask runs on a CSR without the gate or y_accumulate")
    if isinstance(A, PanelCSR):
        if gate_ref is not None:
            raise MMRecError("spmm: the cosine gate needs the whole row sum: not available on a PanelCSR")
        last = len(A.panels) - 1
        for i, P in enumerate(A.panels):                              # Y accumulates over the panels; the running sum takes every
            run_in = None if acc_out is None else (acc_in if i == 0 else acc_out)   # panel's share, the division comes with the last one
            spmm_raw(P, X, Y=Y, acc_in=run_in, acc_out=acc_out, acc_div=acc_div if i == last else 1.0, use_plan=use_plan,
                     y_accumulate=Y is not None and (i > 0 or y_accumulate))
        return
    _need_cuda(X, Y, acc_in, acc_out, gate_ref)
    lib = _lib.load()
    if X.dim() != 2 or X.shape[0] != A.n_cols:
        raise MMRecError(f"spmm: X is {tuple(X.shape)}, matrix has {A.n_cols} columns")
    X = _f32c(X)
    d = X.shape[1]
    for name, t in (("Y", Y), ("acc_in", acc_in), ("acc_out", acc_out), ("gate_ref", gate_ref)):
        if t is not None and (t.shape != (A.n_rows, d) or not t.is_contiguous() or t.dtype != torch.float32):
            raise MMRecError(f"spmm: {name} must be contiguous float32 [{A.n_rows}, {d}]")
    if Y is None and acc_out is None:
        raise MMRecError("spmm: nothing to write")
    if y_accumulate and (gate_ref is not None or Y is None):
        raise MMRecError("spmm: y_accumulate needs Y and no gate")
    if drop is not None:
        keep = drop[0]
        _need_cuda(keep)
        if keep.dtype != torch.int32 or not keep.is_contiguous() or keep.numel() < (A.nnz + 31) // 32:
            raise MMRecError("spmm: keep_bits must be contiguous int32 [ceil(nnz / 32)]")
    op = _spmm_op(A, X, Y=Y, acc_in=acc_in, acc_out=acc_out, acc_div=acc_div, gate_ref=gate_ref, y_accumulate=y_accumulate,
                  drop=drop, use_plan=use_plan)
    check(lib.mmrec_spmm_run_f32(d, 1, ctypes.byref(op), 0, _stream()), "mmrec_spmm_run_f32")


def _spmm_op(A: CSR, X, Y=None, acc_in=None, acc_out=None, acc_div=1.0, gate_ref=None, y_accumulate=False, drop=None, post=None,
             post_row0=0, sync_before=False, use_plan=True):
    """One `mmrec_spmm_op` over A's work plan (none with `use_plan=False` or an empty plan).  X and acc_in are a tensor or a
    (rows below the split, rows from the split on) pair; the other operands have leading dimension d."""
    X_lo, X_hi = X if isinstance(X, tuple) else (X, None)
    in_lo, in_hi = acc_in if isinstance(acc_in, tuple) else (acc_in, None)
    d = X_lo.shape[1]
    op = _lib.SpmmOp(n_rows=A.n_rows, n_cols=A.n_cols, rowptr=_ptr(A.rowptr), colidx=_ptr(A.colidx), vals=_ptr(A.vals),
                     X=_ptr(X_lo), ldx=X_lo.stride(0), Y=_ptr(Y), ldy=d, y_accumulate=int(y_accumulate),
                     acc_in=_ptr(in_lo), acc_out=_ptr(acc_out), ldacc=d, acc_div=float(acc_div), gate_ref=_ptr(gate_ref), ldgate=d,
                     post=_ptr(post), ldpost=d, post_row0=int(post_row0), sync_before=int(bool(sync_before)))
    if use_plan and A.n_tasks > 0:
        op.tasks, op.n_tasks, op.n_cta_tasks = _ptr(A.tasks), A.n_tasks, A.n_cta_tasks
        op.split_rows, op.counters, op.partial = _ptr(A.split_rows), _ptr(A.counters), _ptr(A.partial(d))
    if X_hi is not None:
        op.X_hi, op.ldx_hi, op.x_split = _ptr(X_hi), X_hi.stride(0), X_lo.shape[0]
    if in_hi is not None:
        op.acc_in_hi, op.ldacc_in_hi, op.acc_in_split = _ptr(in_hi), in_hi.stride(0), in_lo.shape[0]
    if drop is not None:
        op.keep_bits, op.keep_scale = _ptr(drop[0]), float(drop[1])
    return op


class _SpmmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, A: CSR, base):
        ctx.A = A
        ctx.has_base = base is not None
        out = torch.empty(A.n_rows, X.shape[1], dtype=torch.float32, device=X.device)
        if base is None:
            spmm_raw(A, X, Y=out)
        else:
            spmm_raw(A, X, acc_in=_f32c(base), acc_out=out)
        return out

    @staticmethod
    def backward(ctx, g):
        g = _f32c(g)
        At = ctx.A.t()
        gx = torch.empty(At.n_rows, g.shape[1], dtype=torch.float32, device=g.device)
        spmm_raw(At, g, Y=gx)                       # dX = A^T dY  (autograd of torch.sparse.mm)
        return gx, None, (g if ctx.has_base else None)


def spmm(A: CSR, X: torch.Tensor, base: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`base + A @ X` (base optional), differentiable w.r.t. X and base."""
    return _SpmmFn.apply(X, A, base)


def propagate_mean_fused(A: CSR, ego, n_layers: int, post_csr: Optional[CSR] = None, post_x: Optional[torch.Tensor] = None,
                         post_layers: int = 1, post_row0: int = 0, cooperative: bool = True) -> torch.Tensor:
    """Inference form of `propagate_mean` (+ FREEDOM / BM3's item-item term) as one `mmrec_spmm_run_f32` call:
    `mean(E_0 .. E_L)`, and if `post_csr` is given `out[post_row0:] += post_csr^post_layers @ post_x`
    (`src/models/freedom.py:164-178`: `h = mm_adj @ ... @ item_emb`, `i_g + h`).  No autograd.

    `ego` is E_0 as one tensor or as the pair (user table, item table): layer 1 then gathers from the two tables and adds
    them to the running sum where they are, bit-identical to propagating their concatenation without making it.
    `cooperative`: all steps in one cooperative launch with grid barriers; otherwise one ordinary launch per group of
    independent steps (the item-item product shares layer 1's launch, each later layer is one launch).  Falls back to one
    launch per SpMM when the chained kernel does not take the shape."""
    pair = isinstance(ego, (tuple, list))
    parts = [_f32c(t) for t in ego] if pair else [_f32c(ego)]
    _need_cuda(*parts, post_x)
    d = parts[0].shape[1]
    n = sum(t.shape[0] for t in parts)
    if pair and any(t.shape[1] != d for t in parts):
        raise MMRecError("propagate_mean_fused: the two tables differ in width")
    if n != A.n_rows or n != A.n_cols:
        raise MMRecError(f"propagate_mean_fused: E_0 has {n} rows, the matrix is {A.n_rows} x {A.n_cols}")
    e0 = tuple(parts) if pair else parts[0]

    def unfused():
        return _propagate_mean_post_unfused(A, torch.cat(parts) if pair else parts[0], n_layers, post_csr, post_x, post_layers, post_row0)

    if n_layers < 1 or A.n_tasks == 0 or (post_csr is not None and post_csr.n_tasks == 0):
        return unfused()
    # wave = how many launch boundaries (or grid barriers) must precede a step: h_i = post_csr @ h_{i-1} waits for h_{i-1},
    # layer l for layer l - 1, and the last layer, whose epilogue adds h, also for the last item-item product
    waves, keep = [], []
    h = None
    if post_csr is not None:
        h = _f32c(post_x)
        for i in range(post_layers):                                 # h = mm_adj @ h, the first one reads the parameters only
            y = torch.empty(post_csr.n_rows, d, dtype=torch.float32, device=parts[0].device)
            waves.append((i, 1, post_csr, dict(X=h, Y=y)))
            keep.append(y)
            h = y
    acc = torch.empty(n, d, dtype=torch.float32, device=parts[0].device)
    x = e0
    for l in range(1, n_layers + 1):
        last = l == n_layers
        y = None if last else torch.empty_like(acc)
        wave = max(l - 1, post_layers) if (last and h is not None) else l - 1
        waves.append((wave, 0, A, dict(X=x, Y=y, acc_in=e0 if l == 1 else acc, acc_out=acc,
                                       acc_div=float(n_layers + 1) if last else 1.0, post=h if last else None, post_row0=post_row0)))
        keep.append(y)
        x = y
    if len(waves) > 8:
        return unfused()
    waves.sort(key=lambda w: (w[0], w[1]))                          # within a wave: the A_hat layer first, the shorter product fills its tail
    arr = (_lib.SpmmOp * len(waves))(*[_spmm_op(M, sync_before=i > 0 and w != waves[i - 1][0], **kw)
                                         for i, (w, _, M, kw) in enumerate(waves)])
    rc = _lib.load().mmrec_spmm_run_f32(d, len(arr), arr, int(cooperative), _stream())
    if rc == -4:                                                     # MMREC_EUNSUPPORTED: shape without a chained kernel
        return unfused()
    check(rc, "mmrec_spmm_run_f32")
    return acc


def _propagate_mean_post_unfused(A, ego, n_layers, post_csr, post_x, post_layers, post_row0):
    out = _PropagateMeanFn.apply(ego.detach(), A, n_layers)
    if post_csr is not None:
        h = _f32c(post_x).detach()
        for _ in range(post_layers - 1):
            y = torch.empty(post_csr.n_rows, h.shape[1], dtype=torch.float32, device=h.device)
            spmm_raw(post_csr, h, Y=y)
            h = y
        tail = out[post_row0:]
        spmm_raw(post_csr, h, acc_in=tail, acc_out=tail)
    return out


class _PropagateMeanFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ego, A: CSR, n_layers: int, drop: Optional[tuple] = None, div: Optional[float] = None):
        # drop = (keep_bits, keep_bits_t, scale) of a symmetric A: the forward multiplies by the dropped matrix, the backward
        # by its transpose, which is the same CSR with the mirrored bits.  div: the divisor of the last epilogue, L + 1 (the
        # layer mean) unless given; 1 gives the plain sum E_0 + ... + E_L
        div = float(n_layers + 1) if div is None else float(div)
        ctx.A, ctx.L, ctx.drop, ctx.div = A, n_layers, drop, div
        ego = _f32c(ego)
        if n_layers == 0:
            return ego.clone()
        fwd = None if drop is None else (drop[0], drop[2])
        acc = torch.empty_like(ego)
        x = ego
        for l in range(1, n_layers + 1):
            last = l == n_layers
            y = None if last else torch.empty_like(ego)
            spmm_raw(A, x, Y=y, acc_in=ego if l == 1 else acc, acc_out=acc, acc_div=div if last else 1.0, drop=fwd)
            x = y
        return acc

    @staticmethod
    def backward(ctx, g):
        L = ctx.L
        gm = _f32c(g) if ctx.div == 1.0 else _f32c(g) / ctx.div      # d out / d E_l, the same for every layer
        if L == 0:
            return g, None, None, None, None
        drop = ctx.drop
        At = ctx.A.t() if drop is None else ctx.A
        bwd = None if drop is None else (drop[1], drop[2])
        cur = gm
        for _ in range(L):                          # g_l = gm + A^T g_{l+1}
            nxt = torch.empty_like(gm)
            spmm_raw(At, cur, acc_in=gm, acc_out=nxt, drop=bwd)
            cur = nxt
        return cur, None, None, None, None


def propagate_mean(A: CSR, ego: torch.Tensor, n_layers: int) -> torch.Tensor:
    """mean(E_0 .. E_L), E_{l+1} = A E_l -- the LightGCN propagation every graph model repeats
    (`src/models/freedom.py:169-176`, `bm3.py:86-92`, `lightgcn.py:116-123`, `mgcn.py:159-166`), with the
    running sum and the final division fused into the SpMM epilogue (no stack, no extra passes)."""
    return _PropagateMeanFn.apply(ego, A, n_layers)


def propagate_sum(A: CSR, ego: torch.Tensor, n_layers: int) -> torch.Tensor:
    """E_0 + E_1 + ... + E_L, E_{l+1} = A E_l: `propagate_mean` with 1 as the final divisor, so the running sum in the
    SpMM epilogue is the whole result.  DualGNN's tower (`src/models/dualgnn.py:311-314`: `h = conv(x)`, `h_1 = conv(h)`,
    `x_hat = h + x + h_1`) is L = 2: the first epilogue forms x + h, the second (x + h) + h_1, the reference's order of
    additions.  Backward: g_l = g + A^T g_{l+1}."""
    return _PropagateMeanFn.apply(ego, A, n_layers, None, 1.0)


def edge_keep_bits(draws: torch.Tensor, keep_prob: float, draw_of: torch.Tensor, mirror: Optional[torch.Tensor] = None):
    """The keep bits of one `sparse_dropout` draw (`src/common/encoders.py:77-84`): `floor(float32(1 - rate) + draws)`
    with one fp32 add, draw j applied to the CSR position e with draw_of[e] = j (`graph.dropout_entry_maps`).  Returns
    (keep_bits, keep_bits_t) as int32 [ceil(nnz / 32)] (bit e of word e // 32); keep_bits_t (None without `mirror`) holds
    bit mirror[e] of keep_bits at e: the transpose of the dropped symmetric matrix on the same CSR."""
    _need_cuda(draws, draw_of, mirror)
    draws = _f32c(draws)
    nnz = draws.numel()
    for name, t in (("draw_of", draw_of), ("mirror", mirror)):
        if t is not None and (t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != nnz):
            raise MMRecError(f"edge_keep_bits: {name} must be contiguous int32 [{nnz}]")
    n_words = (nnz + 31) // 32
    if n_words == 0:                                # nothing to launch: one word of zeros, as "bits past nnz are 0" promises
        keep = torch.zeros(1, dtype=torch.int32, device=draws.device)
        return keep, None if mirror is None else torch.zeros_like(keep)
    keep = torch.empty(n_words, dtype=torch.int32, device=draws.device)
    keep_t = None if mirror is None else torch.empty_like(keep)
    check(_lib.load().mmrec_edge_keep_bits(nnz, _ptr(draws), float(keep_prob), _ptr(draw_of), _ptr(mirror), _ptr(keep), _ptr(keep_t),
                                           _stream()), "mmrec_edge_keep_bits")
    return keep, keep_t


def propagate_mean_dropped(A: CSR, ego: torch.Tensor, n_layers: int, keep: torch.Tensor, keep_t: torch.Tensor,
                           scale: float) -> torch.Tensor:
    """`propagate_mean` through the edge-dropped matrix of SelfCF's encoder (`src/common/encoders.py:90-112`: `sparse_dropout`
    of the normalised adjacency, then `torch.sparse.mm` per layer and the layer mean), on the fixed CSR and its fixed plan:
    the entries whose bit of `keep` is set, weighted fl(v * scale) (`mmrec_spmm_op.keep_bits`).  Differentiable w.r.t. `ego`; the
    backward runs the same CSR with `keep_t` (`edge_keep_bits` with the mirror map), as A is symmetric bit for bit."""
    if not A.symmetric:
        raise MMRecError("propagate_mean_dropped: the backward reads the transpose through the mirrored bits; A must be symmetric")
    _need_cuda(ego, keep, keep_t)
    return _PropagateMeanFn.apply(ego, A, n_layers, (keep, keep_t, float(scale)))


def propagate_layergcn(A: CSR, ego: torch.Tensor, n_layers: int) -> torch.Tensor:
    """Inference form of `src/models/layergcn.py:125-138`: E_{l+1} = cos(A E_l, E_0) * A E_l, sum over layers
    1..L, gate and running sum fused into the SpMM epilogue.  (Training goes through `spmm` + torch ops so
    that autograd sees the cosine gate.)"""
    ego = _f32c(ego)
    if n_layers <= 0:
        return torch.zeros_like(ego)                 # the sum over layers 1..L of nothing
    acc = torch.empty_like(ego)
    x = ego
    for l in range(1, n_layers + 1):
        y = torch.empty_like(ego)
        spmm_raw(A, x, Y=y, acc_in=None if l == 1 else acc, acc_out=acc, gate_ref=ego)
        x = y
    return acc


# ------------------------------------------------------------------------------------------------
# K2: modality projection
# ------------------------------------------------------------------------------------------------
def project_raw(table, weight, bias, idx=None, l2_normalize=False) -> torch.Tensor:
    _need_cuda(table, weight, bias, idx)
    lib = _lib.load()
    table, weight = _f32c(table), _f32c(weight)
    bias = None if bias is None else _f32c(bias)
    if idx is not None:
        idx = idx.to(torch.int64).contiguous()
    n_out = table.shape[0] if idx is None else idx.numel()
    d, F = weight.shape
    if table.shape[1] != F:
        raise MMRecError(f"project: table has {table.shape[1]} features, weight expects {F}")
    out = torch.empty(n_out, d, dtype=torch.float32, device=table.device)
    ws = _ws("project", lib.mmrec_project_workspace_bytes(n_out, F, d), table.device)
    check(lib.mmrec_project_f32(n_out, _ptr(idx), _ptr(table), table.shape[0], F, _ptr(weight), _ptr(bias), d,
                                int(l2_normalize), _ptr(out), d, _ptr(ws), ws.numel(), _stream()), "mmrec_project_f32")
    return out


def set_project_path(tensor_core: bool):
    """True (default): wgmma 3xTF32 projection kernel; False: exact fp32 CUDA-core kernel."""
    _lib.load().mmrec_project_set_path(int(bool(tensor_core)))


# -- f1: backward of the projection and the optimiser step (csrc/train.cu) -------------------------------------------
def index_sum_rows(g: torch.Tensor, idx: torch.Tensor, n_rows: int) -> torch.Tensor:
    """G[i] = sum_{j: idx[j] = i} g[j] in ascending j (`mmrec_index_sum_rows_f32`): `zeros.index_add_(0, idx, g)` made
    bit-reproducible.  The table gradient of a gathered projection is `G @ W` (linearity), so the scatter is d wide."""
    _need_cuda(g, idx)
    g = _f32c(g)
    idx = idx.to(torch.int64).contiguous()
    G = torch.empty(n_rows, g.shape[1], dtype=torch.float32, device=g.device)
    check(_lib.load().mmrec_index_sum_rows_f32(idx.numel(), _ptr(idx), _ptr(g), g.stride(0), g.shape[1], n_rows, _ptr(G), G.stride(0),
                                               _stream()), "mmrec_index_sum_rows_f32")
    return G


def linear_wgrad(g: torch.Tensor, table: torch.Tensor, idx: Optional[torch.Tensor] = None, want_bias: bool = True):
    """(dW [d, F], db [d] | None) of `y = table[idx] @ W^T + b` for the upstream gradient g [n, d]: `g.t().mm(x)`, `g.sum(0)`
    (autograd of `nn.Linear`, src/models/freedom.py:205-209) through `mmrec_linear_wgrad_f32`."""
    _need_cuda(g, table, idx)
    lib = _lib.load()
    g, table = _f32c(g), _f32c(table)
    if idx is not None:
        idx = idx.to(torch.int64).contiguous()
    n, d = g.shape
    F = table.shape[1]
    dW = torch.empty(d, F, dtype=torch.float32, device=g.device)
    db = torch.empty(d, dtype=torch.float32, device=g.device) if want_bias else None
    ws = _ws("wgrad", lib.mmrec_linear_wgrad_workspace_bytes(n, F, d), g.device)
    check(lib.mmrec_linear_wgrad_f32(n, _ptr(idx), _ptr(g), g.stride(0), d, _ptr(table), table.shape[0], F, _ptr(dW), _ptr(db),
                                     _ptr(ws), ws.numel(), _stream()), "mmrec_linear_wgrad_f32")
    return dW, db


def linear_dgrad(G: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """`G @ W` as a fresh [n_rows, F] tensor (`mmrec_linear_dgrad_f32`): the dense table gradient autograd expects."""
    _need_cuda(G, weight)
    G, weight = _f32c(G), _f32c(weight)
    out = torch.empty(G.shape[0], weight.shape[1], dtype=torch.float32, device=G.device)
    check(_lib.load().mmrec_linear_dgrad_f32(G.shape[0], _ptr(G), G.stride(0), G.shape[1], _ptr(weight), weight.shape[1], _ptr(out),
                                             _stream()), "mmrec_linear_dgrad_f32")
    return out


def linear_dgrad_adam(G, weight, param, exp_avg, exp_avg_sq, beta1, beta2, eps, weight_decay, step_size, bc2_sqrt):
    """One Adam step of `param` [n_rows, F] with the gradient `G @ W` computed inside the kernel, never stored
    (`mmrec_linear_dgrad_adam_f32`; torch.optim.Adam.step of src/common/trainer.py:189 fused with the projection backward)."""
    _need_cuda(G, weight, param, exp_avg, exp_avg_sq)
    G, weight = _f32c(G), _f32c(weight)
    for t in (param, exp_avg, exp_avg_sq):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (G.shape[0], weight.shape[1]):
            raise MMRecError("linear_dgrad_adam: param / exp_avg / exp_avg_sq must be contiguous float32 [n_rows, F]")
    check(_lib.load().mmrec_linear_dgrad_adam_f32(G.shape[0], _ptr(G), G.stride(0), G.shape[1], _ptr(weight), weight.shape[1], _ptr(param),
                                                  _ptr(exp_avg), _ptr(exp_avg_sq), float(beta1), float(beta2), float(eps),
                                                  float(weight_decay), float(step_size), float(bc2_sqrt), _stream()),
          "mmrec_linear_dgrad_adam_f32")


def adam_step(entries, beta1, beta2, eps, weight_decay):
    """`entries`: (param, grad, exp_avg, exp_avg_sq, step_size, bc2_sqrt) per tensor; all updated by `mmrec_adam_f32`."""
    import ctypes
    if not entries:
        return
    arr = (_lib.AdamTensor * len(entries))()
    for a, (p, g, m, v, step_size, bc2_sqrt) in zip(arr, entries):
        _need_cuda(p, g, m, v)
        for t in (p, g, m, v):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != p.numel():
                raise MMRecError("adam_step: contiguous float32 tensors of one size per entry")
        a.param, a.grad, a.exp_avg, a.exp_avg_sq, a.n = _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel()
        a.step_size, a.bc2_sqrt = float(step_size), float(bc2_sqrt)
    check(_lib.load().mmrec_adam_f32(len(entries), ctypes.cast(arr, ctypes.c_void_p), float(beta1), float(beta2), float(eps),
                                     float(weight_decay), _stream()), "mmrec_adam_f32")


class _ProjectFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, weight, bias, idx):
        ctx.save_for_backward(table, weight, idx)
        ctx.has_bias = bias is not None
        ctx.table_param = table if isinstance(table, torch.nn.Parameter) else None
        return project_raw(table, weight, bias, idx, False)

    @staticmethod
    def backward(ctx, g):
        # Backward of nn.Linear over the (gathered) table (SURVEY.md 8f f1) on the kernels of csrc/train.cu.
        table, weight, idx = ctx.saved_tensors
        g = _f32c(g)
        gw = gb = gt = None
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            gw, gb = linear_wgrad(g, table, idx, want_bias=ctx.has_bias and ctx.needs_input_grad[2])
            if not ctx.needs_input_grad[1]:
                gw = None
        if ctx.needs_input_grad[0]:
            G = g if idx is None else index_sum_rows(g, idx, table.shape[0])     # d-wide scatter; the table gradient is G @ W
            p = ctx.table_param
            owner = getattr(p, "_mmrec_defer", None) if p is not None else None
            if owner is not None and owner() is not None and getattr(p, "_mmrec_pending", None) is None \
                    and weight.shape[0] <= 128 and weight.shape[1] % 4 == 0:
                # The optimiser (optim.FusedAdam) asked for the gradient in factored form: it updates the table with G @ W
                # computed inside its kernel, so the [n_items, F] gradient never exists.  `.grad` stays None for this table.
                p._mmrec_pending = (G, weight, weight._version)
            else:
                gt = linear_dgrad(G, weight)
        return gt, gw, gb, None


def project(table, weight, bias=None, idx=None, l2_normalize=False) -> torch.Tensor:
    """`Linear(table)[idx]` computed only for the gathered rows (`src/models/freedom.py:205-209`,
    `bm3.py:102-104`, `mgcn.py:148-150`); `l2_normalize` adds `F.normalize` (`mmgcn.py:165-168`)."""
    needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (table, weight, bias))
    if not needs_grad:
        return project_raw(table, weight, bias, idx, l2_normalize)
    y = _ProjectFn.apply(table, weight, bias, idx)
    return torch.nn.functional.normalize(y) if l2_normalize else y


# -- a5b: MGCN's row-wise fusion (csrc/fuse.cu), inference form ---------------------------------------------------------
def gate_rows(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], mul: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`mul * sigmoid(x @ weight.T + bias)` in one kernel (`mmrec_gate_rows_f32`): MGCN's behaviour-guided purifier
    `item_id_embedding.weight * gate_v(image_feats)` (src/models/mgcn.py:153-154).  No autograd."""
    _need_cuda(x, weight, bias, mul, out)
    x, weight = _f32c(x), _f32c(weight)
    n, d = x.shape
    if weight.shape != (d, d):
        raise MMRecError(f"gate_rows: weight must be [{d}, {d}]")
    if bias is not None and bias.shape != (d,):
        raise MMRecError(f"gate_rows: bias must be [{d}], got {tuple(bias.shape)}")
    if mul is not None and mul.shape != (n, d):
        raise MMRecError(f"gate_rows: mul must be [{n}, {d}], got {tuple(mul.shape)}")
    if out is None:
        out = torch.empty(n, d, dtype=torch.float32, device=x.device)
    elif out.shape != (n, d) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != x.device:
        raise MMRecError(f"gate_rows: out must be a contiguous float32 [{n}, {d}] tensor on {x.device}")
    check(_lib.load().mmrec_gate_rows_f32(n, d, _ptr(x), _ptr(weight), _ptr(None if bias is None else _f32c(bias)),
                                          _ptr(None if mul is None else _f32c(mul)), _ptr(out), _stream()), "mmrec_gate_rows_f32")
    return out


def mgcn_fuse(img, txt, content, q_w, q_b, q_w2, gi_w, gi_b, gt_w, gt_b, want_side: bool = False):
    """MGCN's attention over the two modality views, preference gates and `content + side` (src/models/mgcn.py:187-201)
    for all rows in one kernel (`mmrec_mgcn_fuse_f32`).  Returns `all_embeds` (and `side` if asked).  No autograd."""
    _need_cuda(img, txt, content, q_w, q_b, q_w2, gi_w, gi_b, gt_w, gt_b)
    img, txt, content = _f32c(img), _f32c(txt), _f32c(content)
    n, d = img.shape
    if txt.shape != (n, d) or content.shape != (n, d):
        raise MMRecError("mgcn_fuse: img, txt and content must share one shape")
    for name, w in (("q_w", q_w), ("gi_w", gi_w), ("gt_w", gt_w)):
        if w.shape != (d, d):
            raise MMRecError(f"mgcn_fuse: {name} must be [{d}, {d}], got {tuple(w.shape)}")
    for name, b in (("q_b", q_b), ("gi_b", gi_b), ("gt_b", gt_b)):
        if b.shape != (d,):
            raise MMRecError(f"mgcn_fuse: {name} must be [{d}], got {tuple(b.shape)}")
    if q_w2.numel() != d:
        raise MMRecError(f"mgcn_fuse: q_w2 must have {d} elements, got {q_w2.numel()}")
    out = torch.empty(n, d, dtype=torch.float32, device=img.device)
    side = torch.empty_like(out) if want_side else None
    check(_lib.load().mmrec_mgcn_fuse_f32(n, d, _ptr(img), _ptr(txt), _ptr(content), _ptr(_f32c(q_w)), _ptr(_f32c(q_b)),
                                          _ptr(_f32c(q_w2).reshape(-1)), _ptr(_f32c(gi_w)), _ptr(_f32c(gi_b)), _ptr(_f32c(gt_w)),
                                          _ptr(_f32c(gt_b)), _ptr(out), _ptr(side), _stream()), "mmrec_mgcn_fuse_f32")
    return (out, side) if want_side else out


# ------------------------------------------------------------------------------------------------
# K3: scoring, mask, top-k
# ------------------------------------------------------------------------------------------------
def set_score_path(path):
    """"simt" (0): exact fp32 CUDA cores; "tc" (1): wgmma 3xTF32 + mask + radix top-k kernels; "auto" (2, default):
    fused where its shape rules allow, else tc; "fused" (3): wgmma f16 filter with the top-k fused into the GEMM epilogue."""
    if isinstance(path, str):
        path = {"simt": 0, "tc": 1, "auto": 2, "fused": 3}[path]
    _lib.load().mmrec_score_set_path(int(path))


def score(user_e, item_e, users=None) -> torch.Tensor:
    """S = U[users] I^T, freshly allocated fp32 [B, n_items] owned by the caller (the trainer mutates it):
    `torch.matmul(u_embeddings, restore_item_e.transpose(0, 1))` (`src/models/freedom.py:216-220`)."""
    _need_cuda(user_e, item_e, users)
    lib = _lib.load()
    user_e, item_e = _f32c(user_e), _f32c(item_e)
    if users is not None:
        users = users.to(torch.int64).contiguous()
    B = user_e.shape[0] if users is None else users.numel()
    n_items, d = item_e.shape
    out = torch.empty(B, n_items, dtype=torch.float32, device=item_e.device)
    ws = _ws("score", lib.mmrec_score_workspace_bytes(B, n_items, d), item_e.device)
    check(lib.mmrec_score_f32(B, _ptr(users), _ptr(user_e), user_e.stride(0), n_items, _ptr(item_e), item_e.stride(0), d,
                              _ptr(out), n_items, _ptr(ws), ws.numel(), _stream()), "mmrec_score_f32")
    return out


def mask_topk(scores: torch.Tensor, mask: Optional[torch.Tensor], k: int, item_offset: int = 0):
    """`scores[mask[0], mask[1]] = -1e10; torch.topk(scores, k)` (`src/common/trainer.py:307-309`), in place on
    `scores`.  Returns (values, indices); equal scores come out in ascending item index."""
    _need_cuda(scores, mask)
    lib = _lib.load()
    if not (scores.is_contiguous() and scores.dtype == torch.float32 and scores.dim() == 2):
        raise MMRecError("mask_topk: scores must be contiguous float32 [B, n_items]")
    B, n_items = scores.shape
    if mask is not None and mask.numel() > 0:
        mask = mask.to(torch.int64).contiguous()
        check(lib.mmrec_mask_f32(mask.shape[1], _ptr(mask[0]), _ptr(mask[1]), B, n_items, item_offset, _ptr(scores),
                                 n_items, _stream()), "mmrec_mask_f32")
    idx = torch.empty(B, k, dtype=torch.int64, device=scores.device)
    val = torch.empty(B, k, dtype=torch.float32, device=scores.device)
    check(lib.mmrec_topk_rows_f32(B, n_items, _ptr(scores), n_items, k, item_offset, _ptr(idx), _ptr(val), _stream()),
          "mmrec_topk_rows_f32")
    return val, idx


class Catalog:
    """The item side of the scoring contraction prepared once per embedding table (`mmrec_catalog_pack_f32`): fp16
    operand tiles (power-of-two scaled, 11 significand bits) + the maximum row norm of the error bound.  The reference re-reads the same `restore_item_e` for every
    evaluation batch (`src/common/trainer.py:302-310`); a model keeps one Catalog next to its cached evaluation
    embeddings and drops it with them.  Holds a reference to `item_e`: the pair must stay consistent."""

    def __init__(self, item_e: torch.Tensor):
        _need_cuda(item_e)
        lib = _lib.load()
        self.item_e = _f32c(item_e)
        n_items, d = self.item_e.shape
        nbytes = lib.mmrec_catalog_bytes(n_items, d)
        if nbytes == 0:
            raise MMRecError(f"catalog: no tensor-core path for d = {d}")
        self.buf = torch.empty(nbytes + 1024, dtype=torch.uint8, device=item_e.device)
        self.ptr = (self.buf.data_ptr() + 1023) // 1024 * 1024
        check(lib.mmrec_catalog_pack_f32(n_items, _ptr(self.item_e), self.item_e.stride(0), d, self.ptr, nbytes, _stream()),
              "mmrec_catalog_pack_f32")


def score_topk(user_e, item_e, users, mask, k: int, item_offset: int = 0, out=None, catalog: Optional[Catalog] = None):
    """Fused `full_sort_predict` + mask + top-k (`src/models/freedom.py:216-220` + `src/common/trainer.py:304-309`)
    without materialising the [B, n_items] score matrix in HBM.  Returns (values [B,k], indices int64 [B,k]); `out` =
    (values, indices) buffers to write into (e.g. peer-mapped memory in the sharded evaluation); `catalog` = the
    `Catalog` of exactly this `item_e` (else the item operand is packed inside the call)."""
    _need_cuda(user_e, item_e, users, mask)
    lib = _lib.load()
    user_e, item_e = _f32c(user_e), _f32c(item_e)
    if catalog is not None and (catalog.item_e.data_ptr() != item_e.data_ptr() or catalog.item_e.shape != item_e.shape):
        raise MMRecError("score_topk: the catalog was packed from a different item table")
    if users is not None:
        users = users.to(torch.int64).contiguous()
    B = user_e.shape[0] if users is None else users.numel()
    n_items, d = item_e.shape
    if out is not None:
        val, idx = out
        assert val.shape == (B, k) and idx.shape == (B, k) and val.dtype == torch.float32 and idx.dtype == torch.int64 \
            and val.is_contiguous() and idx.is_contiguous()
    else:
        idx = torch.empty(B, k, dtype=torch.int64, device=item_e.device)
        val = torch.empty(B, k, dtype=torch.float32, device=item_e.device)
    m0 = m1 = None
    nnz = 0
    if mask is not None and mask.numel() > 0:
        mask = mask.to(torch.int64).contiguous()
        m0, m1, nnz = mask[0], mask[1], mask.shape[1]
    nbytes = lib.mmrec_score_topk_workspace_bytes(B, n_items, d, k) + 4 * nnz + 4096
    ws = _ws("score_topk", nbytes, item_e.device)
    _last_fused.update(ws=ws, args=(B, n_items, d, k, nnz, int(catalog is None)))
    check(lib.mmrec_score_topk_cat_f32(B, _ptr(users), _ptr(user_e), user_e.stride(0), n_items, _ptr(item_e),
                                       item_e.stride(0), d, None if catalog is None else catalog.ptr, nnz, _ptr(m0), _ptr(m1), k,
                                       item_offset, _ptr(idx), _ptr(val), _ptr(ws), ws.numel(), _stream()), "mmrec_score_topk_cat_f32")
    return val, idx


class _MaxDotFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, t):
        val, idx = score_topk(q, t, None, None, 1)
        val, idx = val.view(-1), idx.view(-1)
        ctx.save_for_backward(q, t, idx)
        ctx.mark_non_differentiable(idx)
        return val, idx

    @staticmethod
    def backward(ctx, g, _g_idx):
        # the gradient of a max reaches the selected pair only: O(B d), no [B, M] or [B, M, d] tensor
        q, t, idx = ctx.saved_tensors
        g = _f32c(g).unsqueeze(1)
        dq = g * t[idx] if ctx.needs_input_grad[0] else None
        dt = index_sum_rows(g * q, idx, t.shape[0]) if ctx.needs_input_grad[1] else None
        return dq, dt


def max_dot(q: torch.Tensor, t: torch.Tensor):
    """`torch.max(torch.sum(q[:, None, :] * t[None, :, :], -1), dim=-1)` without the [B, M, d] product or the [B, M] scores:
    MVGAE's hardest in-batch negative (`src/models/mvgae.py:73-85`, which builds `z[users.repeat(1, B)] * z[neg_items]`).
    q [B, d] and t [M, d] are fp32 device tensors.  Returns (values [B], index int64 [B]): values[b] is the largest
    `<q_b, t_j>` in the fp32 chain of `score_topk` (K3, k = 1), index[b] the lowest j that reaches it.  Only `values` is
    differentiable: dq = g t[index], dt = index_sum_rows(g q, index, M) (contributions to a row of t summed in ascending b,
    so the gradient is bit-reproducible).  Memory: O(B d) per call; the scratch is `score_topk`'s cached workspace, shared
    with the evaluation and bounded (its unfused route's score block is capped at 64 MiB).

    NaN: the chain's NaN is the positive canonical NaN, which K3's key order ranks above +inf, and equal keys go to the
    lowest index; so a row with a NaN score returns NaN at its first NaN column, as `torch.max` does (whatever the sign
    bit of the NaN that went into q or t).  Scores are never -0.0 (the chain starts from +0.0), so +0.0 and -0.0 never
    compete."""
    _need_cuda(q, t)
    if q.dim() != 2 or t.dim() != 2 or q.shape[1] != t.shape[1] or t.shape[0] < 1:
        raise MMRecError(f"max_dot: q {tuple(q.shape)} and t {tuple(t.shape)} must be [B, d] and [M >= 1, d]")
    return _MaxDotFn.apply(q, t)


_last_fused: dict = {}


def fused_fallback_rows(*_ignored) -> int:
    """Diagnostic (synchronises): how many rows of the last row block of the last fused score_topk call went through the
    exact fp32 kernel; -1 when that call did not take the fused path."""
    _refuse_capture("fused_fallback_rows")
    if not _last_fused:
        return -1
    return int(_lib.load().mmrec_debug_fused_fallback_rows(_ptr(_last_fused["ws"]), *_last_fused["args"]))


def fused_stage_times():
    """Tuning aid: device microseconds of the stages of the last fused score_topk call (env MMREC_CF_TIMING must be set
    before the first call): [catalogue pack, prep + mask, pass 1, threshold, pass 2, finalists, exact rows]."""
    import ctypes
    buf = (ctypes.c_float * 16)()
    n = _lib.load().mmrec_debug_cf_timing(ctypes.cast(buf, ctypes.c_void_p), 16)
    return [float(buf[i]) for i in range(n)]


def knn_topk(x: torch.Tensor, k: int, rows: Optional[torch.Tensor] = None, norms: Optional[torch.Tensor] = None,
             shrink: Optional[float] = None):
    """Top-k of `x[rows] @ x.T` per query row (all rows by default) without the [m, n] similarity matrix
    (`mmrec_knn_topk_f32`, K7): the cosine kNN of `src/models/freedom.py:79-91` / `src/utils/utils.py:165-172` for the
    normalised feature table `x`.  Returns (values [m, k], indices int64 [m, k]), bit-identical to `score(x[rows], x)`
    followed by `mask_topk(.., None, k)` on the CUDA-core path.

    With `shrink` (`mmrec_knn_topk_shrink_f32`): ranked by `(x[q] . x[i]) / (norms[q] * norms[i] + shrink)`, ItemKNNCBF's
    `build_item_sim_matrix` (`src/models/itemknncbf.py:56-65`); `norms` defaults to `torch.norm(x, p=2, dim=-1)`, the
    reference's expression.  Bit-identical to the score, that elementwise denominator, then `mask_topk(.., None, k)`.

    Synchronises (it reads back how many rows take the exact route): refused while the stream captures a CUDA graph."""
    _refuse_capture("knn_topk")
    _need_cuda(x, rows, norms)
    lib = _lib.load()
    if x.dim() != 2:
        raise MMRecError("knn_topk: x must be [n, F]")
    x = _f32c(x)
    n, F = x.shape
    if rows is not None:
        rows = rows.to(torch.int64).contiguous()
        if rows.dim() != 1:
            raise MMRecError("knn_topk: rows must be 1-D")
        if rows.numel() and (int(rows.min()) < 0 or int(rows.max()) >= n):
            raise MMRecError(f"knn_topk: rows outside [0, {n})")
    m = n if rows is None else rows.numel()
    if not (1 <= k <= min(1024, n)):
        raise MMRecError(f"knn_topk: need 1 <= k <= min(1024, n = {n}), got {k}")
    idx = torch.empty(m, k, dtype=torch.int64, device=x.device)
    val = torch.empty(m, k, dtype=torch.float32, device=x.device)
    if m == 0:
        return val, idx
    ws = _ws("knn", lib.mmrec_knn_topk_workspace_bytes(n, F, m, k) + 1024, x.device)
    if shrink is None:
        check(lib.mmrec_knn_topk_f32(n, _ptr(x), x.stride(0), F, m, _ptr(rows), k, _ptr(idx), _ptr(val), _ptr(ws), ws.numel(),
                                     _stream()), "mmrec_knn_topk_f32")
    else:
        norms = torch.norm(x, p=2, dim=-1) if norms is None else _f32c(norms)
        if norms.shape != (n,):
            raise MMRecError(f"knn_topk: norms must be [{n}]")
        check(lib.mmrec_knn_topk_shrink_f32(n, _ptr(x), x.stride(0), F, m, _ptr(rows), k, _ptr(norms), float(shrink), _ptr(idx),
                                            _ptr(val), _ptr(ws), ws.numel(), _stream()), "mmrec_knn_topk_shrink_f32")
    # the graphs are built once, at model construction: the scratch (2 n F bytes of fp16 pack) is not kept for later calls
    # (the call has synchronised the stream, so the memory is free to go back to the allocator)
    _ws_cache.pop(("knn", x.device.index, torch.cuda.current_stream(x.device).cuda_stream), None)
    return val, idx


def knn_fallback_rows() -> int:
    """Diagnostic: rows of the last `knn_topk` call that took the exact route (all of them when the table held a
    non-finite element); -1 before the first call."""
    _refuse_capture("knn_fallback_rows")
    return int(_lib.load().mmrec_debug_knn_fallback_rows())


# ------------------------------------------------------------------------------------------------
# K9: user scores from the sparse interactions and the sparse item kNN graph (ItemKNNCBF)
# ------------------------------------------------------------------------------------------------
def _sparse_pair(R: CSR, S: CSR, users):
    if R.n_cols != S.n_rows or S.n_rows != S.n_cols:
        raise MMRecError(f"sparse scores: R [{R.n_rows}, {R.n_cols}] and S [{S.n_rows}, {S.n_cols}] do not chain")
    _need_cuda(R.rowptr, S.rowptr, users)
    if users is not None:
        users = users.to(torch.int64).contiguous()
    return users, (R.rowptr, R.colidx, _f32c(R.vals), S.rowptr, S.colidx, _f32c(S.vals))


def sparse_scores(R: CSR, S: CSR, users: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Rows `users` of `R @ S` as a fresh dense fp32 [B, n_items] owned by the caller (the trainer mutates it):
    `self.scores_matrix[user]` with `scores_matrix = torch.mm(r_matrix, item_sim)` (`src/models/itemknncbf.py:54`,
    `:107-111`), summed per element over R's row in ascending column order (`mmrec_sparse_scores_f32`, K9)."""
    users, parts = _sparse_pair(R, S, users)
    B = R.n_rows if users is None else users.numel()
    out = torch.empty(B, S.n_cols, dtype=torch.float32, device=R.rowptr.device)
    check(_lib.load().mmrec_sparse_scores_f32(B, _ptr(users), S.n_cols, *(_ptr(t) for t in parts), _ptr(out), S.n_cols, _stream()),
          "mmrec_sparse_scores_f32")
    return out


def sparse_score_topk(R: CSR, S: CSR, users: Optional[torch.Tensor], mask: Optional[torch.Tensor], k: int):
    """Fused `sparse_scores` + `scores[mask[0], mask[1]] = -1e10` + top-k (`src/common/trainer.py:304-309`) without a
    dense row (`mmrec_sparse_score_topk_f32`, K9).  Returns (values [B, k], indices int64 [B, k]), bit-identical to
    `mask_topk(sparse_scores(R, S, users), mask, k)`.

    Synchronises (it reads back how many rows take the unfused route): refused while the stream captures a CUDA graph."""
    _refuse_capture("sparse_score_topk")
    users, parts = _sparse_pair(R, S, users)
    _need_cuda(mask)
    lib = _lib.load()
    B = R.n_rows if users is None else users.numel()
    n_items = S.n_cols
    if not (1 <= k <= min(1024, n_items)):
        raise MMRecError(f"sparse_score_topk: need 1 <= k <= min(1024, n_items = {n_items}), got {k}")
    m0 = m1 = None
    nnz = 0
    if mask is not None and mask.numel() > 0:
        mask = mask.to(torch.int64).contiguous()
        m0, m1, nnz = mask[0], mask[1], mask.shape[1]
    dev = R.rowptr.device
    idx = torch.empty(B, k, dtype=torch.int64, device=dev)
    val = torch.empty(B, k, dtype=torch.float32, device=dev)
    ws = _ws("sparse_topk", lib.mmrec_sparse_score_topk_workspace_bytes(B, n_items, nnz, k), dev)
    check(lib.mmrec_sparse_score_topk_f32(B, _ptr(users), n_items, *(_ptr(t) for t in parts), nnz, _ptr(m0), _ptr(m1), k, _ptr(idx),
                                          _ptr(val), _ptr(ws), ws.numel(), _stream()), "mmrec_sparse_score_topk_f32")
    return val, idx


def sparse_topk_fallback_rows() -> int:
    """Diagnostic: rows of the last `sparse_score_topk` call served by the unfused route (too many products or masked
    items for shared memory, or a non-finite score); -1 before the first call."""
    _refuse_capture("sparse_topk_fallback_rows")
    return int(_lib.load().mmrec_debug_sparse_topk_fallback_rows())


# ------------------------------------------------------------------------------------------------
# K8: full-table exp-sum (LGMRec's hypergraph contrastive loss)
# ------------------------------------------------------------------------------------------------
def _expsum_args(q, t):
    _need_cuda(q, t)
    if q.dim() != 2 or t.dim() != 2 or q.shape[1] != t.shape[1]:
        raise MMRecError(f"expsum_rows: q {tuple(q.shape)} and t {tuple(t.shape)} must be [B, d] and [M, d]")
    if q.shape[1] not in (32, 64, 128):
        raise MMRecError(f"expsum_rows: d must be 32, 64 or 128, got {q.shape[1]}")
    return _f32c(q), _f32c(t)


class _ExpsumRowsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, t, inv_tau: float):
        q, t = _expsum_args(q, t)
        ctx.save_for_backward(q, t)
        ctx.inv_tau = inv_tau
        lib = _lib.load()
        (B, d), M = q.shape, t.shape[0]
        ttl = torch.empty(B, dtype=torch.float32, device=q.device)
        ws = _ws("expsum", lib.mmrec_expsum_rows_workspace_bytes(B, M, d), q.device)
        check(lib.mmrec_expsum_rows_f32(B, _ptr(q), q.stride(0), M, _ptr(t), t.stride(0), d, inv_tau, _ptr(ttl), _ptr(ws), ws.numel(),
                                        _stream()), "mmrec_expsum_rows_f32")
        return ttl

    @staticmethod
    def backward(ctx, g):
        q, t = ctx.saved_tensors
        want_q, want_t = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (want_q or want_t):
            return None, None, None
        lib = _lib.load()
        g = _f32c(g)
        (B, d), M = q.shape, t.shape[0]
        dq = torch.empty_like(q) if want_q else None
        dt = torch.empty_like(t) if want_t else None
        ws = _ws("expsum", lib.mmrec_expsum_rows_workspace_bytes(B, M, d), q.device)
        check(lib.mmrec_expsum_rows_bwd_f32(B, _ptr(q), q.stride(0), M, _ptr(t), t.stride(0), d, ctx.inv_tau, _ptr(g), _ptr(dq), d,
                                            _ptr(dt), d, _ptr(ws), ws.numel(), _stream()), "mmrec_expsum_rows_bwd_f32")
        return dq, dt, None


def expsum_rows(q: torch.Tensor, t: torch.Tensor, tau: float) -> torch.Tensor:
    """`torch.exp(torch.matmul(q, t.T) / tau).sum(dim=1)` (`src/models/lgmrec.py:164`, the `ttl_score` of `ssl_triple_loss`)
    without the [B, M] matrix, in the forward and in the backward (`mmrec_expsum_rows_f32` / `_bwd_f32`, K8), with
    gradients for q and t.  d must be 32, 64 or 128."""
    return _ExpsumRowsFn.apply(q, t, 1.0 / float(tau))


def topk_merge(vals: torch.Tensor, idx: torch.Tensor):
    """Merge per-shard top-k lists [parts, B, k] into the global top-k [B, k] (SURVEY.md 8e eval collective)."""
    _need_cuda(vals, idx)
    lib = _lib.load()
    vals, idx = _f32c(vals), idx.to(torch.int64).contiguous()
    parts, B, k = vals.shape
    out_i = torch.empty(B, k, dtype=torch.int64, device=vals.device)
    out_v = torch.empty(B, k, dtype=torch.float32, device=vals.device)
    check(lib.mmrec_topk_merge(parts, B, k, _ptr(vals), _ptr(idx), _ptr(out_i), _ptr(out_v), _stream()), "mmrec_topk_merge")
    return out_v, out_i


def _ptr_array(ptrs):
    import ctypes
    arr = (ctypes.c_void_p * len(ptrs))(*[int(x) for x in ptrs])
    return arr, ctypes.cast(arr, ctypes.c_void_p)


def topk_merge_peers(val_ptrs, idx_ptrs, B, k, device, idx_mul=1, idx_add=0, row0=0, n_rows=None, sync=None):
    """`topk_merge` over lists left where each rank wrote them: raw device addresses of `parts` [B, k] value (fp32) and
    index (int64) lists, rank order; index -> idx * idx_mul + part * idx_add (round-robin shards: world, 1).  Rows
    [row0, row0 + n_rows) only (default: all): returns ([n_rows, k] values, indices).  `sync` = (flag_ptrs, state, rank):
    the ranks are synchronised inside the kernel (before the lists are read) instead of by a barrier launch."""
    lib = _lib.load()
    n_rows = B - row0 if n_rows is None else n_rows
    va, vap = _ptr_array(val_ptrs)
    ia, iap = _ptr_array(idx_ptrs)
    out_i = torch.empty(n_rows, k, dtype=torch.int64, device=device)
    out_v = torch.empty(n_rows, k, dtype=torch.float32, device=device)
    fa = fap = None
    if sync is not None:
        fa, fap = _ptr_array(sync[0])
    check(lib.mmrec_topk_merge_peers(len(val_ptrs), B, k, vap, iap, int(idx_mul), int(idx_add), int(row0), int(n_rows), _ptr(out_i),
                                     _ptr(out_v), fap, None if sync is None else _ptr(sync[1]), 0 if sync is None else int(sync[2]),
                                     _stream()), "mmrec_topk_merge_peers")
    return out_v, out_i


def peer_sum(part_ptrs, n, acc_in=None, acc_out=None, acc_div=1.0, sum_out=None):
    """K4: `sum_out = sum_r parts[r]` (rank order), `acc_out = (acc_in + sum) / acc_div` -- the user-embedding exchange of
    the item-sharded propagation as one pass over peer-mapped buffers (`part_ptrs`: raw device addresses, rank order)."""
    lib = _lib.load()
    arr, arrp = _ptr_array(part_ptrs)
    check(lib.mmrec_peer_sum_f32(int(n), len(part_ptrs), arrp, _ptr(acc_in), _ptr(acc_out), float(acc_div),
                                 _ptr(sum_out), _stream()), "mmrec_peer_sum_f32")
    return sum_out, acc_out


def peer_reduce_push(part_ptrs, dst_ptrs, n, rank, acc_in=None, acc_out=None, acc_div=1.0, final_layer=False):
    """K4, reduce-scatter + all-gather form (`mmrec_peer_reduce_push_f32`): this rank sums ITS slice of all partials and
    stores the result (final layer: `(acc + sum) / acc_div`) into that slice of every rank's destination buffer;
    `acc_in` / `acc_out` hold this rank's slice of the running layer sum."""
    lib = _lib.load()
    pa, pap = _ptr_array(part_ptrs)
    da, dap = _ptr_array(dst_ptrs)
    check(lib.mmrec_peer_reduce_push_f32(int(n), len(part_ptrs), int(rank), pap, dap, _ptr(acc_in), _ptr(acc_out), float(acc_div),
                                         int(bool(final_layer)), _stream()), "mmrec_peer_reduce_push_f32")


def peer_exchange(part_ptrs, dst_ptrs, flag_ptrs, state, n, rank, acc_in=None, acc_out=None, acc_div=1.0, final_layer=False):
    """`peer_reduce_push` with both rank synchronisations inside the kernel (`mmrec_peer_exchange_f32`): one launch per layer."""
    lib = _lib.load()
    pa, pap = _ptr_array(part_ptrs)
    da, dap = _ptr_array(dst_ptrs)
    fa, fap = _ptr_array(flag_ptrs)
    check(lib.mmrec_peer_exchange_f32(int(n), len(part_ptrs), int(rank), pap, dap, fap, _ptr(state), _ptr(acc_in), _ptr(acc_out),
                                      float(acc_div), int(bool(final_layer)), _stream()), "mmrec_peer_exchange_f32")


def peer_barrier(flag_ptrs, state, rank):
    """Device-side barrier of the ranks on the current stream over the same flags (`mmrec_peer_barrier`)."""
    fa, fap = _ptr_array(flag_ptrs)
    check(_lib.load().mmrec_peer_barrier(len(flag_ptrs), int(rank), fap, _ptr(state), _stream()), "mmrec_peer_barrier")


def peer_gather(src_ptrs, n_each, dst: torch.Tensor):
    """`dst[p * n_each + i] = src[p][i]`: all-gather of a sharded table by peer loads (`mmrec_peer_gather_f32`)."""
    lib = _lib.load()
    sa, sap = _ptr_array(src_ptrs)
    check(lib.mmrec_peer_gather_f32(int(n_each), len(src_ptrs), sap, _ptr(dst), _stream()), "mmrec_peer_gather_f32")
    return dst


def topk_metric_sums(topk_idx: torch.Tensor, pos_ptr: torch.Tensor, pos_items: torch.Tensor, disc: torch.Tensor, idcg_all: torch.Tensor,
                     sums: torch.Tensor):
    """f2: adds, per position j < K, the sum over the rows of `topk_idx` of recall / ndcg / precision / map at j + 1 to `sums`
    [4, K] float64 (`mmrec_topk_metrics_f64`; src/utils/topk_evaluator.py:70-102 + src/utils/metrics.py:12-105 on the device)."""
    _need_cuda(topk_idx, pos_ptr, pos_items, disc, idcg_all, sums)
    lib = _lib.load()
    n, K = topk_idx.shape
    assert topk_idx.dtype == torch.int64 and topk_idx.is_contiguous() and pos_ptr.dtype == torch.int64 and pos_items.dtype == torch.int64
    assert sums.dtype == torch.float64 and sums.shape == (4, K) and sums.is_contiguous() and disc.dtype == torch.float64
    check(lib.mmrec_topk_metrics_f64(n, K, _ptr(topk_idx), _ptr(pos_ptr), _ptr(pos_items), _ptr(disc), _ptr(idcg_all), _ptr(sums),
                                     _stream()), "mmrec_topk_metrics_f64")
    return sums


def bipartite_norm(users: torch.Tensor, items: torch.Tensor, n_users: int, n_items: int, eps: float = 1e-7) -> torch.Tensor:
    """fp32 1/sqrt((d_u+eps)(d_i+eps)) per edge, as `_normalize_adj_m` (`src/models/freedom.py:145-154`)."""
    _need_cuda(users, items)
    lib = _lib.load()
    users, items = users.to(torch.int64).contiguous(), items.to(torch.int64).contiguous()
    vals = torch.empty(users.numel(), dtype=torch.float32, device=users.device)
    ws = _ws("bnorm", lib.mmrec_bipartite_norm_workspace_bytes(n_users, n_items), users.device)
    check(lib.mmrec_bipartite_norm_f32(users.numel(), _ptr(users), _ptr(items), n_users, n_items, eps, _ptr(vals), _ptr(ws),
                                       ws.numel(), _stream()), "mmrec_bipartite_norm_f32")
    return vals
