"""MGCN's fusion kernels (a5b), the edge norms (K1c) and K8's strided and misaligned load / store paths, element by element.

Until these tests, a5b was checked by one Frobenius norm per tensor and K8 only on contiguous, aligned tables.  Here:

* a5b pre-activations.  Each of `gate_rows_kernel`'s and `mgcn_fuse_kernel`'s pre-activations is a sequential chain
  acc = b_j (+0 without a bias), acc = fmaf(W[j, k], x_k, acc) for k = 0 .. d-1, restated by `oracle.fuse_chain_f32`
  with a correctly rounded fmaf.  A wrong bias slot, a wrong `jt`, a dropped k or a row of the persistent grid's second
  sweep is then a wrong bit.
* `gate_rows` bit for bit.  The epilogue `g = 1 / (1 + expf(-acc))`, `out = mul * g` is applied to the emulated chain on
  the device with torch in fp32.  ASSUMPTION: torch's CUDA `exp` is CUDA's `expf` and its `/` is IEEE division
  (neither PyTorch nor this library is built with fast math).  `test_gate_rows_sigmoid_alone` reads the kernel's
  sigmoid with nothing else in play (one-hot rows, no bias: acc = W[j, k] exactly), so it fails first if this
  assumption ever breaks.
* `mgcn_fuse` per element.  The four chains (query on img and on txt, both preference gates) are emulated in fp32; the
  rest is evaluated in fp64 from them and each element of `out` and `side` is held to a worst-case bound propagated
  operation by operation (`_Err`).  For a computed x~ = x + dx with |dx| <= ex:
      add / sub   |fl(x~ + y~) - (x + y)| <= ex + ey + u (|x| + |y| + ex + ey)
      mul         |fl(x~ y~) - x y|       <= |x| ey + |y| ex + ex ey + u (|x| + ex)(|y| + ey)
      div         |fl(x~ / y~) - x / y|   <= (ex |y| + |x| ey) / (|y| (|y| - ey)) + u (|x| + ex) / (|y| - ey)
      expf, tanhf <= 2 ulp (CUDA Math API, Table 8): |f~(x~) - f(x)| <= L ex + 2^-22 (|f(x)| + L ex) + 2^-148,
                  L = the largest |f'| on [x - ex, x + ex] (e^(x + ex) for exp, 1 for tanh)
      the logit   sum_j fmaf(w2_j, tanh_j, .) over a lane's d / 32 terms, then 5 butterfly additions: at most
                  d / 32 + 5 roundings on any path, so |err| <= sum_j |w2_j| e_tanh_j + gamma_(d/32 + 5) sum_j |w2_j| (|tanh_j| + e_tanh_j)
  with u = 2^-24, one rounding per remaining operation.  Each bound sums the magnitudes of the operands, so it holds
  under cancellation (`cont + side` near 0) and whichever of the two logits the kernel takes as its maximum (both
  branches are bounded where the logits are too close to tell).  The combine is not pinned bit for bit: nvcc may
  contract `w0 * ximg + w1 * xtxt` and `sep_i + sep_t` into FMAs, which only removes roundings the bound allows for.
* Rows: zeros, saturating pre-activations (|acc| ~ 100s), a NaN row (stays confined to its row), equal logits (weights
  exactly 1/2) and logits more than 104 apart (the smaller view's expf is 0, its weight exactly 0); n from 1 to past two
  sweeps of the persistent grid, S = SMs x warps x 4 rows (warps = 8 for d <= 64, 4 for d = 128).
* Edge norms: `oracle.bipartite_norm_f32` is the kernel's four IEEE operations per side, bit for bit, with degrees
  above 2^24 (where the int -> float conversion rounds) and nodes without edges.
* K8 (`mmrec_expsum_rows_f32` / `_bwd_f32` through the C ABI): leading dimensions > d, a base one float off 16-byte
  alignment (the scalar-load branch) and padded gradient outputs must give the contiguous call's bits (every output is
  a fixed sequence of fp32 operations), leaving the padding untouched.  One exact case does not rest on the kernel's
  error bound: Q rows are -2^7 on a few columns (tf32 lo = 0), T rows positive with 13 significant bits (tf32 lo != 0),
  so every <q, t> is exactly 0 (disjoint supports, e = 1) or <= -256 / inv_tau (e = +0).  ttl is then a count, and
  dQ, dT are exact integer sums (asserted below 2^22 units by `oracle.assert_exact_matmul`; ASSUMPTION as in
  tests/test_gpu_exact_arith.py: the tensor cores' adder keeps >= 24 significant bits), scaled by one rounding for dQ.
  With lo on T in dQ and on P = e g in dT, a missing lo.hi or hi.lo wgmma is a wrong integer.
"""
import numpy as np
import pytest
import torch

from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ULP2 = 2.0 ** -22                 # 2 ulp of an fp32 value, relative
TINY = 2.0 ** -148                # 2 ulp of the smallest subnormal


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _sweep_rows(d):
    """S: rows one sweep of the persistent grid covers (fuse.cu: one CTA per SM, warps x 4 rows each)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * (8 if d <= 64 else 4) * 4


def _n_rows(spec, d):
    S = _sweep_rows(d)
    return {"S-1": S - 1, "S": S, "S+1": S + 1, "2S+5": 2 * S + 5}.get(spec, spec)


N_SPECS = [1, 3, 4, 5, "S-1", "S", "S+1", "2S+5"]


def _linear(rng, d_out, d_in, scale=1.0):
    a = scale / np.sqrt(d_in)
    return rng.uniform(-a, a, (d_out, d_in)).astype(np.float32), rng.uniform(-a, a, d_out).astype(np.float32)


# ======================================================================================================================
# a5b: gate_rows
# ======================================================================================================================
_GATE = {}


def _gate_case(d):
    """Rows for the largest n (prefixes serve the smaller ones) and their emulated chains, with and without the bias."""
    if d not in _GATE:
        S = _sweep_rows(d)
        N = 2 * S + 5
        rng = np.random.default_rng(d)
        W, b = _linear(rng, d, d)
        X = rng.standard_normal((N, d)).astype(np.float32)
        X[1] = 0.0                                                      # zeros: acc = b
        X[3] *= np.float32(300.0)                                       # |acc| in the hundreds: g = 0 or 1
        X[S] *= np.float32(-300.0)
        X[2] = np.nan                                                   # NaN confined to its row
        X[S - 1] = np.nan
        mul = rng.standard_normal((N, d)).astype(np.float32)
        _GATE[d] = (W, b, X, mul, O.fuse_chain_f32(X, W, b), O.fuse_chain_f32(X, W, None))
    return _GATE[d]


def _gate_epilogue(acc, mul):
    """The kernel's epilogue, on the device in fp32: g = 1 / (1 + expf(-acc)), out = mul * g."""
    g = torch.div(torch.ones_like(acc), torch.exp(-acc) + 1.0)
    return g if mul is None else mul * g


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("n_spec", N_SPECS)
def test_gate_rows_bit_exact(dev, d, n_spec):
    from mmrec_b200 import ops
    W, b, X, mul, acc_b, acc_0 = _gate_case(d)
    n = _n_rows(n_spec, d)
    Wd, bd, Xd, Md = (torch.from_numpy(a).to(dev) for a in (W, b, X[:n], mul[:n]))
    A_b, A_0 = torch.from_numpy(acc_b[:n]).to(dev), torch.from_numpy(acc_0[:n]).to(dev)
    O.assert_bits(ops.gate_rows(Xd, Wd, bd, mul=Md), _gate_epilogue(A_b, Md), f"d={d} n={n} bias, mul")
    O.assert_bits(ops.gate_rows(Xd, Wd, None), _gate_epilogue(A_0, None), f"d={d} n={n} no bias, no mul")
    O.assert_bits(ops.gate_rows(Xd, Wd, None, mul=Md), _gate_epilogue(A_0, Md), f"d={d} n={n} no bias, mul")
    # out= a row slice of a larger tensor, as MGCN passes emb[U:]
    big = torch.full((n + 9, d), 7.0, device=dev)
    ret = ops.gate_rows(Xd, Wd, bd, out=big[5:5 + n])
    assert ret.data_ptr() == big[5].data_ptr()
    O.assert_bits(big[5:5 + n], _gate_epilogue(A_b, None), f"d={d} n={n} out= view")
    assert bool((big[:5] == 7.0).all()) and bool((big[5 + n:] == 7.0).all())
    got = ops.gate_rows(Xd, Wd, bd, mul=Md).cpu()
    nan_rows = torch.isnan(got).any(1).nonzero().flatten().tolist()
    S = _sweep_rows(d)
    assert nan_rows == [r for r in (2, S - 1) if r < n] and all(bool(torch.isnan(got[r]).all()) for r in nan_rows)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_gate_rows_sigmoid_alone(dev, d):
    """One-hot rows without a bias: acc[k, j] = W[j, k] exactly, so the output is the kernel's sigmoid of W^T."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(100 + d)
    W = (rng.standard_normal((d, d)) * 8).astype(np.float32)           # spans the saturated ends too
    Wd = torch.from_numpy(W).to(dev)
    got = ops.gate_rows(torch.eye(d, device=dev), Wd, None)
    O.assert_bits(got, _gate_epilogue(Wd.t().contiguous(), None), f"d={d} sigmoid of W^T")


# ======================================================================================================================
# a5b: mgcn_fuse
# ======================================================================================================================
class _Err:
    """A value computed in fp32 by the kernel, as (exact value in fp64, bound on |computed - exact|)."""

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, np.float64)

    def __add__(self, o):
        return _Err(self.v + o.v, self.e + o.e + U * (abs(self.v) + abs(o.v) + self.e + o.e))

    def __neg__(self):
        return _Err(-self.v, self.e)

    def __sub__(self, o):
        return self + (-o)

    def __mul__(self, o):
        return _Err(self.v * o.v, abs(self.v) * o.e + abs(o.v) * self.e + self.e * o.e + U * (abs(self.v) + self.e) * (abs(o.v) + o.e))

    def __truediv__(self, o):
        den = abs(o.v) - o.e
        assert not (den <= 0).any()
        return _Err(self.v / o.v, (self.e * abs(o.v) + abs(self.v) * o.e) / (abs(o.v) * den) + U * (abs(self.v) + self.e) / den)

    def exp(self):
        v = np.exp(self.v)
        lip_e = np.exp(self.v) * np.expm1(self.e)
        return _Err(v, lip_e + ULP2 * (v + lip_e) + TINY)


def _sigmoid(x):
    """1 / (1 + expf(-x)).  Where expf may overflow to inf the kernel's result is 0, off by at most the exact value."""
    one = _Err(np.ones_like(x.v))
    e = (-x).exp()
    g = one / (one + e)
    return _Err(g.v, g.e + np.where(e.v + e.e >= 2.0 ** 127, g.v, 0.0))


def _fuse_bound(hi, ht, gi, gt, w2, img, txt, cont):
    """fp64 values and error bounds of `side` and `out` from the kernel's exact fp32 chains (see the module docstring)."""
    d = img.shape[1]
    w2 = w2.astype(np.float64)
    gam = (d // 32 + 5) * U / (1 - (d // 32 + 5) * U)

    def logit(h):
        t = np.tanh(h.astype(np.float64))
        et = ULP2 * abs(t) + TINY
        return _Err((w2 * t).sum(1), (abs(w2) * et).sum(1) + gam * (abs(w2) * (abs(t) + et)).sum(1))

    si, st = logit(hi), logit(ht)

    def weights(s_max, s_other):                                       # m = s_max: e_max = 1 exactly
        one = _Err(np.ones_like(s_max.v))
        e = (s_other - s_max).exp()
        den = one + e
        return one / den, e / den

    a0, a1 = weights(si, st)                                           # w0, w1 when the kernel's max is si
    b1, b0 = weights(st, si)                                           # ... when it is st
    sure_i = si.v - st.v > si.e + st.e
    sure_t = st.v - si.v > si.e + st.e
    with np.errstate(invalid="ignore"):
        w0 = _Err(np.where(sure_t, b0.v, a0.v), np.where(sure_i, a0.e, np.where(sure_t, b0.e, np.maximum(a0.e, b0.e))))
        w1 = _Err(np.where(sure_t, b1.v, a1.v), np.where(sure_i, a1.e, np.where(sure_t, b1.e, np.maximum(a1.e, b1.e))))
    col = lambda x: _Err(x.v[:, None], x.e[:, None])                   # noqa: E731
    xi, xt, xc = _Err(img), _Err(txt), _Err(cont)
    common = col(w0) * xi + col(w1) * xt
    side = (_sigmoid(_Err(gi)) * (xi - common) + _sigmoid(_Err(gt)) * (xt - common) + common) / _Err(np.full_like(img, 3.0, np.float64))
    return side, xc + side


_FUSE = {}


def _fuse_case(d):
    if d not in _FUSE:
        S = _sweep_rows(d)
        N = 2 * S + 5
        rng = np.random.default_rng(1000 + d)
        qw, qb = _linear(rng, d, d)
        giw, gib = _linear(rng, d, d)
        gtw, gtb = _linear(rng, d, d)
        s = rng.choice(np.array([-1.0, 1.0], np.float32), d)
        w2 = (s * rng.uniform(2.0, 3.0, d)).astype(np.float32)         # sum |w2| >= 2 d: saturated views are > 104 apart
        img, txt, cont = (rng.standard_normal((N, d)).astype(np.float32) for _ in range(3))

        def view_at(target):                                           # x with qw x + qb = target (so tanh = +-1)
            return np.linalg.solve(qw.astype(np.float64), target - qb.astype(np.float64)).astype(np.float32)

        img[1] = txt[1] = cont[1] = 0.0                                 # zeros
        img[2] = np.nan                                                 # NaN: the whole row, no other
        txt[3] = img[3]                                                 # equal logits: w0 = w1 = 1/2
        img[4], txt[4] = view_at(50.0 * np.sign(w2)), view_at(-50.0 * np.sign(w2))   # logits > 104 apart
        img[5], txt[5] = txt[4], img[4]
        cont[6] *= np.float32(300.0)                                    # saturated gates
        img[7] *= np.float32(300.0)                                     # saturated tanh
        cont[S - 1] = np.nan
        img[S], txt[S] = img[4], txt[4]
        txt[S + 1] = img[S + 1]
        chains = [O.fuse_chain_f32(img, qw, qb), O.fuse_chain_f32(txt, qw, qb), O.fuse_chain_f32(cont, giw, gib),
                  O.fuse_chain_f32(cont, gtw, gtb)]
        _FUSE[d] = ((qw, qb, w2[None, :], giw, gib, gtw, gtb), (img, txt, cont), chains)
    return _FUSE[d]


_WORST = {}


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("n_spec", N_SPECS)
def test_mgcn_fuse_per_element_bound(dev, d, n_spec):
    from mmrec_b200 import ops
    weights, views, chains = _fuse_case(d)
    n = _n_rows(n_spec, d)
    img, txt, cont = (v[:n] for v in views)
    hi, ht, gi, gt = (c[:n] for c in chains)
    out, side = ops.mgcn_fuse(*(torch.from_numpy(v).to(dev) for v in (img, txt, cont)),
                              *(torch.from_numpy(w).to(dev) for w in weights), want_side=True)
    out, side = out.cpu().double().numpy(), side.cpu().double().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        want_side, want_out = _fuse_bound(hi, ht, gi, gt, weights[2][0], img, txt, cont)
    nan_rows = np.isnan(img).any(1) | np.isnan(txt).any(1) | np.isnan(cont).any(1)
    for name, got, want in (("side", side, want_side), ("out", out, want_out)):
        assert np.array_equal(np.isnan(got), np.repeat(nan_rows[:, None], d, 1)), f"{name}: NaN outside the NaN rows"
        ok = ~nan_rows
        err, bound = np.abs(got[ok] - want.v[ok]), want.e[ok] * (1 + 2.0 ** -20)
        assert np.isfinite(bound).all()
        ratio = float((err / np.maximum(bound, 1e-300)).max(initial=0.0))
        _WORST[(name, d)] = max(_WORST.get((name, d), 0.0), ratio)
        if not (err <= bound).all():
            i = np.argmax(err - bound)
            pytest.fail(f"d={d} n={n} {name}: {(err > bound).sum()} elements beyond the bound; worst {err.flat[i]:.3e} > {bound.flat[i]:.3e}")
    print(f"d={d} n={n}: worst error / bound so far {_WORST}")


def test_mgcn_fuse_far_logits_weight_is_zero(dev):
    """Logits more than 104 apart: the kernel's common view is exactly the larger view (weight 1 and 0), so with the gates
    saturated to 0 (content x 300 against the gate weights) side = common / 3 = that view / 3, bit for bit."""
    from mmrec_b200 import ops
    d = 64
    weights, views, _ = _fuse_case(d)
    qw, qb, w2, giw, gib, gtw, gtb = weights
    img, txt = views[0][[4, 5]], views[1][[4, 5]]
    zero_gate = np.zeros_like(gib) - np.float32(1000.0)                 # sigmoid(-1000) = 0 exactly
    cont = np.zeros_like(img)
    args = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (img, txt, cont, qw, qb, w2, giw, zero_gate, gtw, zero_gate)]
    out, side = ops.mgcn_fuse(*args, want_side=True)
    want = (img / np.float32(3.0)).astype(np.float32)                  # row 4: img wins (w0 = 1); row 5: img is the loser
    want[1] = (txt[1] / np.float32(3.0)).astype(np.float32)
    O.assert_bits(side, want, "side with weights 1 / 0")
    O.assert_bits(out, want, "out = 0 + side")


# ======================================================================================================================
# a5b: argument checks
# ======================================================================================================================
def _gate_args(dev, n=6, d=32):
    z = lambda *s: torch.zeros(*s, device=dev)                         # noqa: E731
    return dict(x=z(n, d), weight=z(d, d), bias=z(d), mul=z(n, d), out=z(n, d))


@pytest.mark.parametrize("bad", ["bias_len", "bias_2d", "mul_shape", "out_shape", "out_strided", "out_f64"])
def test_gate_rows_rejects_bad_arguments(dev, bad):
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    a = _gate_args(dev)
    a.update({"bias_len": dict(bias=torch.zeros(31, device=dev)), "bias_2d": dict(bias=torch.zeros(1, 32, device=dev)),
              "mul_shape": dict(mul=torch.zeros(5, 32, device=dev)), "out_shape": dict(out=torch.zeros(7, 32, device=dev)),
              "out_strided": dict(out=torch.zeros(6, 64, device=dev)[:, ::2]),
              "out_f64": dict(out=torch.zeros(6, 32, device=dev, dtype=torch.float64))}[bad])
    with pytest.raises(MMRecError):
        ops.gate_rows(a["x"], a["weight"], a["bias"], mul=a["mul"], out=a["out"])
    ops.gate_rows(**_gate_args(dev))                                   # the well-formed call passes


@pytest.mark.parametrize("bad", ["q_w", "q_b", "q_w2", "gi_w", "gi_b", "gt_w", "gt_b"])
def test_mgcn_fuse_rejects_bad_weight_shapes(dev, bad):
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    n, d = 6, 32
    z = lambda *s: torch.zeros(*s, device=dev)                         # noqa: E731
    w = dict(q_w=z(d, d), q_b=z(d), q_w2=z(1, d), gi_w=z(d, d), gi_b=z(d), gt_w=z(d, d), gt_b=z(d))
    ops.mgcn_fuse(z(n, d), z(n, d), z(n, d), **w)                       # the well-formed call passes
    w[bad] = {"q_w": z(d, d - 1), "q_b": z(d + 1), "q_w2": z(1, d - 1), "gi_w": z(d - 1, d), "gi_b": z(d - 1), "gt_w": z(d, 2 * d),
              "gt_b": z(1)}[bad]
    with pytest.raises(MMRecError):
        ops.mgcn_fuse(z(n, d), z(n, d), z(n, d), **w)


# ======================================================================================================================
# K1c: edge norms
# ======================================================================================================================
def test_bipartite_norm_bit_exact(dev):
    """Degrees from 1 to above 2^24 (2^24 + 3 rounds to 2^24 + 4 in fp32, 2^24 + 1 to 2^24), and nodes without edges."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(7)
    n_users, n_items = 1000, 5000
    hub_u, hub_i = (1 << 24) + 3, (1 << 24) + 1
    users = np.concatenate([np.zeros(hub_u, np.int64), rng.integers(1, n_users - 2, hub_i + 200000)])
    items = np.concatenate([rng.integers(0, n_items - 2, hub_u), np.full(hub_i, 7, np.int64), rng.integers(0, n_items - 2, 200000)])
    p = rng.permutation(users.size)
    users, items = users[p], items[p]
    du, di = np.bincount(users, minlength=n_users), np.bincount(items, minlength=n_items)
    assert du[0] == hub_u and di[7] >= hub_i and du.min() == 0 and di.min() == 0 and (du[1:-2] >= 1).all()
    assert float(np.float32(du[0])) != du[0]
    got = ops.bipartite_norm(torch.from_numpy(users).to(dev), torch.from_numpy(items).to(dev), n_users, n_items)
    O.assert_bits(got, O.bipartite_norm_f32(users, items, n_users, n_items), "bipartite_norm")


# ======================================================================================================================
# K8: strided, misaligned and padded operands through the C ABI
# ======================================================================================================================
def _es_plan(nX, nY):
    from test_gpu_lgmrec import _plan
    return _plan(nX, nY)


def _es_call(dev, B, M, d, q, ldq, t, ldt, inv_tau, g, dq, lddq, dt, lddt):
    """ttl into a fresh tensor, dQ / dT into the given addresses (raw pointers and leading dimensions)."""
    from mmrec_b200 import _lib
    lib = _lib.load()
    nbytes = lib.mmrec_expsum_rows_workspace_bytes(B, M, d)
    ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
    ttl = torch.empty(B, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mmrec_expsum_rows_f32(B, q, ldq, M, t, ldt, d, inv_tau, ttl.data_ptr(), ws.data_ptr(), ws.numel(), st), "fwd")
    _lib.check(lib.mmrec_expsum_rows_bwd_f32(B, q, ldq, M, t, ldt, d, inv_tau, g.data_ptr(), dq, lddq, dt, lddt, ws.data_ptr(),
                                             ws.numel(), st), "bwd")
    return ttl


def _padded(dev, a, ld, shift, fill=float("nan")):
    """a [n, d] copied into a buffer of rows of `ld` floats starting `shift` floats in; returns (buffer, view, address)."""
    n, d = a.shape
    buf = torch.full((n * ld + shift + 8,), fill, device=dev)
    v = buf[shift:shift + n * ld].view(n, ld)
    v[:, :d] = a
    return buf, v, buf.data_ptr() + 4 * shift


ES_SHAPES = [(300, 50), (50, 300), (200, 3000)]          # dQ direct / dT partials, the reverse, both partials


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("B,M", ES_SHAPES)
def test_expsum_strided_and_misaligned_match_contiguous(dev, d, B, M):
    plans = (_es_plan(B, M)[0], _es_plan(M, B)[0])
    assert {(300, 50): (1, 5), (50, 300): (5, 1), (200, 3000): (24, 4)}[(B, M)] == plans
    gen = torch.Generator(device="cuda").manual_seed(d + B)
    q = torch.nn.functional.normalize(torch.randn(B, d, generator=gen, device=dev))
    t = torch.nn.functional.normalize(torch.randn(M, d, generator=gen, device=dev))
    g = torch.rand(B, generator=gen, device=dev) * 2 - 1
    inv_tau = 5.0
    dq0, dt0 = torch.empty(B, d, device=dev), torch.empty(M, d, device=dev)
    ttl0 = _es_call(dev, B, M, d, q.data_ptr(), d, t.data_ptr(), d, inv_tau, g, dq0.data_ptr(), d, dt0.data_ptr(), d)
    for ld_in, shift in ((d + 3, 1), (d + 4, 0)):                      # scalar loads (odd base), vector loads with ld > d
        qb, _, qp = _padded(dev, q, ld_in, shift)                       # the buffers stay referenced: the kernel sees raw addresses
        tb, _, tp = _padded(dev, t, ld_in, shift)
        dqb, dqv, dqp = _padded(dev, torch.full((B, d), float("nan"), device=dev), d + 5, shift)
        dtb, dtv, dtp = _padded(dev, torch.full((M, d), float("nan"), device=dev), d + 5, shift)
        ttl = _es_call(dev, B, M, d, qp, ld_in, tp, ld_in, inv_tau, g, dqp, d + 5, dtp, d + 5)
        what = f"d={d} B={B} M={M} ld={ld_in} shift={shift}"
        O.assert_bits(ttl, ttl0, f"{what} ttl")
        O.assert_bits(dqv[:, :d], dq0, f"{what} dQ")
        O.assert_bits(dtv[:, :d], dt0, f"{what} dT")
        assert bool(torch.isnan(qb[:shift]).all() and torch.isnan(tb[:shift]).all())
        for buf, v in ((dqb, dqv), (dtb, dtv)):                         # padding and the rest of the buffer untouched
            keep = torch.ones_like(buf, dtype=torch.bool)
            keep[shift:shift + v.numel()].view_as(v)[:, :d] = False
            assert bool(torch.isnan(buf[keep]).all()), f"{what}: padding written"


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("B,M", [(2048, 3000), (64, 3000), (3000, 64)])
def test_expsum_exact_integer_case(dev, d, B, M):
    rng = np.random.default_rng(d * 7 + B)
    tau, inv_tau = 0.25, 4.0
    Qi = np.zeros((B, d), np.int64)                                    # -1 on two columns per row (units 2^7)
    for b in range(B):
        Qi[b, rng.choice(d, 2, replace=False)] = -1
    Ti = O.exact_ints(rng, (M, d), 13, density=0.78, signed=False, full=True)   # units 2^-13, 13 significant bits
    gi = O.exact_ints(rng, (B,), 13, full=True)                         # units 2^-13
    q, t = O.to_f32_exact(Qi, 2.0 ** 7), O.to_f32_exact(Ti, 2.0 ** -13)
    g = O.to_f32_exact(gi, 2.0 ** -13)
    assert (O.tf32_split_rn(t)[1][Ti != 0] != 0).all() and (O.tf32_split_rn(g)[1] != 0).all()
    S = O.int_matmul(-Qi, Ti.T)                                         # -<q, t> in units 2^-6
    E = (S == 0).astype(np.int64)                                       # disjoint supports: e = 1 exactly
    assert (S[S != 0] * 2.0 ** -6 * inv_tau >= 130).all()               # the others: e = expf(<= -130) = 0
    assert 0 < E.mean() < 0.2
    O.assert_exact_matmul(E, Ti)                                        # dQ's sums over j
    O.assert_exact_matmul((E * gi[:, None]).T, Qi)                      # dT's sums over b
    want_ttl = E.sum(1).astype(np.float32)
    sq = O.to_f32_exact(O.int_matmul(E, Ti), 2.0 ** -13)                # exact sum_j e t_j
    want_dq = (sq * (np.float32(inv_tau) * g)[:, None]).astype(np.float32)   # one rounding
    want_dt = O.to_f32_exact(O.int_matmul((E * gi[:, None]).T, Qi), 2.0 ** (7 - 13 + 2))   # inv_tau = 2^2: exact
    from mmrec_b200 import ops
    qd = torch.from_numpy(q).to(dev).requires_grad_(True)
    td = torch.from_numpy(t).to(dev).requires_grad_(True)
    ttl = ops.expsum_rows(qd, td, tau)
    ttl.backward(torch.from_numpy(g).to(dev))
    what = f"d={d} B={B} M={M}"
    O.assert_bits(ttl, want_ttl, f"{what} ttl")
    O.assert_bits(qd.grad, want_dq, f"{what} dQ")
    O.assert_bits(td.grad, want_dt, f"{what} dT")
