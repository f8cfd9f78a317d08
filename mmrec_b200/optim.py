"""f1: the optimiser step of the reference's trainer on the kernels of csrc/train.cu.

`FusedAdam` is a drop-in for the `optim.Adam(params, lr=.., weight_decay=..)` the reference's trainer builds
(`src/common/trainer.py:117-118`, stepped at `:189`): the same constructor arguments, `param_groups`, state
names (`step`, `exp_avg`, `exp_avg_sq`) and `state_dict` layout -- it IS a `torch.optim.Adam` whose `step` runs

* `mmrec_adam_f32`: one launch for all ordinary parameters (torch's `_multi_tensor_adam` arithmetic), and
* `mmrec_linear_dgrad_adam_f32` for the trainable modality tables (`nn.Embedding.from_pretrained(v_feat, freeze=False)`,
  `src/models/freedom.py:58,61`): `ops.project`'s backward leaves their gradient in factored form `(G, W)` with
  `grad = G @ W`, and the kernel updates table, exp_avg and exp_avg_sq with that product computed on the fly -- the dense
  [n_items, F] gradient (115 MB per modality at Amazon-baby size) is never written or read.

The factored step reads the table column strip by column strip, which streams HBM less efficiently than the dense route
(`mmrec_linear_dgrad_f32` writing the gradient, then `mmrec_adam_f32` streaming everything linearly; compare with
tools/bench_train.py).  So `factored` is opt-in (`FusedAdam(..., factored=True)` or env MMREC_FACTORED_TABLE_GRAD=1): it trades time for not
holding the [n_items, F] gradient.  The factored form is only used where it is exact: a second backward before `step()` (gradient accumulation), a
gradient from another path, `clip_grad_norm_` or a `weight` that changed since the backward make the pending product
materialise into `.grad` (`materialize_pending`) and the table takes the ordinary route.  There is no CPU path.
"""
from __future__ import annotations

import os
import weakref

import torch

from . import ops
from ._lib import MMRecError


def _bump_version(p):
    """The kernels write through raw pointers, which autograd's version counter does not see; consumers keyed on it (the
    models' evaluation cache, autograd's saved-tensor check) must notice the update."""
    setter = getattr(torch._C._autograd, "_unsafe_set_version_counter", None)
    if setter is not None:
        setter((p,), (p._version + 1,))
    else:
        p.add_(0)


FACTORED_DEFAULT = os.environ.get("MMREC_FACTORED_TABLE_GRAD", "0") == "1"


class FusedAdam(torch.optim.Adam):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, factored=None):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, foreach=False)
        self.factored = FACTORED_DEFAULT if factored is None else bool(factored)
        for group in self.param_groups:
            for p in group["params"]:
                p._mmrec_defer = weakref.ref(self) if self.factored else None   # ops._ProjectFn.backward may leave this parameter's gradient factored
                                                     # for as long as this optimiser lives (`release()` ends it earlier)
                p._mmrec_pending = None

    def release(self):
        """Stop asking for factored gradients (call before handing the parameters to another optimiser)."""
        self.materialize_pending()
        for group in self.param_groups:
            for p in group["params"]:
                p._mmrec_defer = None

    # -- factored gradients ------------------------------------------------------------------------
    @staticmethod
    def _materialize(p):
        pend = getattr(p, "_mmrec_pending", None)
        if pend is None:
            return
        G, weight, version = pend
        p._mmrec_pending = None
        if weight._version != version:
            raise MMRecError("FusedAdam: the projection weight changed between backward and step; the factored table gradient is stale")
        dense = ops.linear_dgrad(G, weight)
        p.grad = dense if p.grad is None else p.grad.add_(dense)

    def materialize_pending(self):
        """Turn every factored table gradient into an ordinary `.grad` (needed before `clip_grad_norm_` or any other
        consumer of `.grad`)."""
        for group in self.param_groups:
            for p in group["params"]:
                self._materialize(p)

    def zero_grad(self, set_to_none: bool = True):
        for group in self.param_groups:
            for p in group["params"]:
                p._mmrec_pending = None
        super().zero_grad(set_to_none=set_to_none)

    # -- step ------------------------------------------------------------------------------------------
    def _state_of(self, p):
        st = self.state[p]
        if len(st) == 0:                        # as torch/optim/adam.py `_init_group`
            st["step"] = torch.tensor(0.0, dtype=torch.float32)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work = []
        for group in self.param_groups:
            if group.get("amsgrad") or group.get("maximize"):
                raise MMRecError("FusedAdam: amsgrad / maximize are not part of the reference's trainer and have no kernel")
            beta1, beta2 = group["betas"]
            lr, eps, wd = float(group["lr"]), group["eps"], group["weight_decay"]
            tables, plain = [], []
            for p in group["params"]:
                pend = getattr(p, "_mmrec_pending", None)
                if pend is not None and (p.grad is not None or pend[1]._version != pend[2] or not p.is_contiguous()):
                    self._materialize(p)
                    pend = None
                if pend is None and p.grad is None:
                    continue
                if p.dtype != torch.float32 or (p.grad is not None and p.grad.is_sparse):
                    raise MMRecError("FusedAdam: dense float32 parameters only")
                st = self._state_of(p)
                st["step"] += 1
                t = float(st["step"])
                bc1, bc2 = 1.0 - beta1 ** t, 1.0 - beta2 ** t
                step_size, bc2_sqrt = (lr / bc1) * -1.0, bc2 ** 0.5          # torch/optim/adam.py, `_multi_tensor_adam`
                (tables if pend is not None else plain).append((p, st, step_size, bc2_sqrt, pend))
            work.append((beta1, beta2, eps, wd, tables, plain))
        # all tables first: their update reads the projection weights of the forward, which the plain pass is about to change
        for beta1, beta2, eps, wd, tables, _ in work:
            for p, st, step_size, bc2_sqrt, (G, weight, _v) in tables:
                ops.linear_dgrad_adam(G, weight, p.data, st["exp_avg"], st["exp_avg_sq"], beta1, beta2, eps, wd, step_size, bc2_sqrt)
                p._mmrec_pending = None
                _bump_version(p)
        for beta1, beta2, eps, wd, _, plain in work:
            entries = []
            for p, st, step_size, bc2_sqrt, _ in plain:
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                if not (p.is_contiguous() and st["exp_avg"].is_contiguous() and st["exp_avg_sq"].is_contiguous()):
                    raise MMRecError("FusedAdam: parameters and their state must be contiguous")
                entries.append((p.data, g, st["exp_avg"], st["exp_avg_sq"], step_size, bc2_sqrt))
            ops.adam_step(entries, beta1, beta2, eps, wd)
            for p, *_ in plain:
                _bump_version(p)
        return loss
