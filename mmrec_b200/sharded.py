"""Item-sharded hot path over N GPUs (one process per GPU, torch.distributed / NCCL over NVLink) -- SURVEY.md 8(e).

The reference has no multi-GPU code at all (`src/utils/configurator.py:114-118` picks one device); the
partitioning follows BASELINE.json's north star: shard the ITEM axis.

  * rank g owns the items {i : i mod N == g} (round-robin, so the Zipf head does not land on one rank), relabelled
    to a contiguous local range; it holds their embeddings, and the column block R_g = R[:, I_g] of the
    interaction matrix as two CSRs (users x local items, and its transpose) with the GLOBAL degree normalisation
    of `get_norm_adj_mat` (`src/models/freedom.py:102-126`);
  * one UI layer:  items   E'_Ig = R_g^T E_U              -- local SpMM, needs the full user table
                   users   E'_U  = sum_g R_g E_Ig         -- local SpMM, then ONE all-reduce of the [U, d] partial
    (= the reduce-scatter + all-gather of user embeddings the north star names);
  * eval: every rank scores all users against its item shard with the fused score+mask+top-k kernel, the
    [B, k] (value, global index) lists are all-gathered and merged by `mmrec_topk_merge` (per-user top-k
    all-reduce).

`spmm` / `score_topk` / `merge` are injectable so that the orchestration + collectives can be exercised on CPU
under gloo (tests/test_sharded_gloo.py); the defaults are this library's CUDA kernels.
"""
from __future__ import annotations

import json
import os
import time

import numpy as np
import torch
import torch.distributed as dist


class ItemShard:
    """Host-side partition of the bipartite training graph for one rank (numpy only)."""

    def __init__(self, inter_row, inter_col, n_users, n_items, rank, world):
        r = np.asarray(inter_row, dtype=np.int64)
        c = np.asarray(inter_col, dtype=np.int64)
        from .graph import unique_sorted
        key = unique_sorted(r * n_items + c)
        r, c = key // n_items, key % n_items
        self.rank, self.world, self.n_users, self.n_items = rank, world, n_users, n_items
        assert n_items < 2 ** 31, "item ids travel as int32 in the top-k exchange"
        self.local_items = np.arange(rank, n_items, world, dtype=np.int64)     # global ids of my items, ascending
        self.n_local = len(self.local_items)
        # global degrees + 1e-7, float64, exactly as the single-GPU builder (freedom.py:113-116)
        du = np.bincount(r, minlength=n_users).astype(np.float64) + 1e-7
        di = np.bincount(c, minlength=n_items).astype(np.float64) + 1e-7
        mine = (c % world) == rank
        self.u = r[mine]
        self.i_local = c[mine] // world
        self.val = ((np.power(du[self.u], -0.5) * 1.0) * np.power(di[c[mine]], -0.5)).astype(np.float32)
        self.nnz = int(mine.sum())

    def to_global(self, local_idx):
        return local_idx * self.world + self.rank

    def mm_coo(self, row, col, val):
        """This rank's rows of an item-item matrix (global COO, e.g. FREEDOM's mm_adj) with LOCAL row ids and RANK-MAJOR
        column ids: global item j sits at (j % world) * n_local + j // world, the layout `mmrec_peer_gather_f32` (or an
        all-gather of the shards) produces.  Needs equally sized shards.  Host only (numpy)."""
        if self.n_items % self.world:
            raise ValueError("mm_coo: n_items must be a multiple of the world size (equal shards)")
        row, col = np.asarray(row, dtype=np.int64), np.asarray(col, dtype=np.int64)
        mine = (row % self.world) == self.rank
        return row[mine] // self.world, (col[mine] % self.world) * self.n_local + col[mine] // self.world, np.asarray(val, dtype=np.float32)[mine]

    def mm_csr(self, row, col, val, device, d=64, l2_bytes=1 << 62):
        """`mm_coo` as a device CSR (duplicates summed, as `coalesce()` does for FREEDOM's mm_adj, freedom.py:74)."""
        from .ops import CSR
        r, c, v = self.mm_coo(row, col, val)
        rt, ct, vt = torch.from_numpy(r).to(device), torch.from_numpy(c).to(device), torch.from_numpy(v).to(device)
        n_cols = self.world * self.n_local
        if n_cols * d * 4 > l2_bytes:
            from .ops import PanelCSR
            return PanelCSR.from_coo(rt, ct, vt, self.n_local, n_cols, d, sum_duplicates=True)
        return CSR.from_coo(rt, ct, vt, self.n_local, n_cols, sum_duplicates=True)

    def csrs(self, device, d=64, l2_bytes=1 << 62):
        """(users x local items, local items x users) as device CSRs; a matrix whose dense operand ([n_cols, d] fp32) is
        larger than `l2_bytes` comes as a column-panelled `ops.PanelCSR`.  (Off by default: every panel re-reads and
        re-writes the whole output for a handful of non-zeros per row.)"""
        from .ops import CSR, PanelCSR
        u = torch.from_numpy(self.u).to(device)
        i = torch.from_numpy(self.i_local).to(device)
        v = torch.from_numpy(self.val).to(device)

        def build(r, c, n_rows, n_cols):
            if n_cols * d * 4 > l2_bytes:
                return PanelCSR.from_coo(r, c, v, n_rows, n_cols, d, sum_duplicates=False)
            return CSR.from_coo(r, c, v, n_rows, n_cols, sum_duplicates=False)
        return build(u, i, self.n_users, self.n_local), build(i, u, self.n_local, self.n_users)


def _cuda_spmm(A, X, acc_in=None, acc_div=1.0, want_y=True):
    from . import ops
    Y = torch.empty(A.n_rows, X.shape[1], dtype=torch.float32, device=X.device) if want_y else None
    acc = None
    if acc_in is not None:
        acc = acc_in
        ops.spmm_raw(A, X, Y=Y, acc_in=acc_in, acc_out=acc, acc_div=acc_div)
    else:
        ops.spmm_raw(A, X, Y=Y)
    return Y, acc


def propagate_mean_sharded(a_ui, a_iu, user_emb, item_emb_local, n_layers, spmm=_cuda_spmm, group=None):
    """mean over layers 0..L of the LightGCN propagation, item-sharded.  Returns (users [U,d] replicated,
    items [I_local,d]).  Per layer: 2 local SpMMs + one all-reduce of the user partial."""
    eu, ei = user_emb, item_emb_local
    acc_u = user_emb.clone()
    acc_i = item_emb_local.clone()
    for l in range(1, n_layers + 1):
        last = l == n_layers
        div = float(n_layers + 1) if last else 1.0
        part_u, _ = spmm(a_ui, ei)                                   # R_g E_Ig : partial user sums
        work = dist.all_reduce(part_u, op=dist.ReduceOp.SUM, group=group, async_op=True)
        ei_next, acc_i = spmm(a_iu, eu, acc_in=acc_i, acc_div=div, want_y=not last)    # overlaps the all-reduce
        work.wait()
        acc_u = acc_u + part_u
        if last:
            acc_u = acc_u / div
        eu, ei = part_u, ei_next
    return acc_u, acc_i


def mm_layer_sharded(shard: ItemShard, mm_local, item_emb_local, i_acc, spmm=_cuda_spmm, group=None):
    """The item-item layer of the sharded FREEDOM in the NCCL / gloo formulation: all-gather of the layer-0 item rows
    (rank-major, what `ItemShard.mm_csr` indexes), then `i_g + mm_adj @ E_I` locally (`src/models/freedom.py:166-167,178`)."""
    world = shard.world
    allrows = torch.empty(world * shard.n_local, item_emb_local.shape[1], dtype=item_emb_local.dtype, device=item_emb_local.device)
    dist.all_gather_into_tensor(allrows, item_emb_local.contiguous(), group=group)
    _, out = spmm(mm_local, allrows, acc_in=i_acc, acc_div=1.0, want_y=False)
    return out


class PeerExchange:
    """Buffers that every rank has mapped (torch symmetric memory: CUDA IPC over NVLink) plus the device-side barrier
    between the ranks' streams.  One allocation, fp32 words:
        parts[l]  [U, d]   this rank's partial user sums of layer l+1 (written by its user-side SpMM)
        gath[l]   [U, d]   the reduced user table of layer l+1: every slice is stored here by the rank that owns it
        items     [I_local, d]  this rank's layer-0 item embeddings (read by the peers for the item-item layer)
        top-k lists  values fp32 [rows, k], indices int64 [rows, k]
    `PeerExchange.create` returns None when this torch build / box cannot provide it -- the caller then keeps the NCCL
    formulation."""

    def __init__(self, hdl, buf, n_users, d, n_layers, n_local, rank, world, topk_rows, k):
        self.hdl, self.buf, self.n, self.rank, self.world = hdl, buf, n_users * d, rank, world
        self.n_layers, self.k, self.topk_rows, self.n_users, self.d, self.n_local = n_layers, k, topk_rows, n_users, d, n_local
        n = self.n
        self.parts = [buf[l * n:(l + 1) * n].view(n_users, d) for l in range(n_layers)]
        self.part_ptrs = [[int(p) + 4 * l * n for p in hdl.buffer_ptrs] for l in range(n_layers)]
        g0 = n_layers * n
        self.gath = [buf[g0 + l * n: g0 + (l + 1) * n].view(n_users, d) for l in range(n_layers)]
        self.gath_ptrs = [[int(p) + 4 * (g0 + l * n) for p in hdl.buffer_ptrs] for l in range(n_layers)]
        i0 = 2 * n_layers * n
        self.items = buf[i0: i0 + n_local * d].view(n_local, d)
        self.item_ptrs = [int(p) + 4 * i0 for p in hdl.buffer_ptrs]
        # top-k lists of the evaluation (8-byte alignment of the index region: every offset before it is even)
        self.val_off = i0 + n_local * d + ((n_local * d) & 1)
        self.idx_off = self.val_off + topk_rows * k + ((topk_rows * k) & 1)
        # this rank's slice of the running layer sum (mmrec_peer_reduce_push_f32: per float4 elements)
        n4 = n // 4
        self.per4 = (n4 + world - 1) // world
        self.lo = min(self.per4 * rank, n4) * 4
        self.hi = min(self.lo + self.per4 * 4, n)
        self.acc = torch.empty(self.per4 * 4, dtype=torch.float32, device=buf.device)
        self._chan = 0
        # flags of the in-kernel barriers (mmrec_peer_exchange_f32 & co): 2 * world ints per rank at the end of the buffer,
        # and this rank's call counter / release word / block counter in ordinary device memory
        self.flag_off = self.idx_off + 2 * topk_rows * k
        self.flag_ptrs = [int(p) + 4 * self.flag_off for p in hdl.buffer_ptrs]
        self.state = torch.zeros(4, dtype=torch.int32, device=buf.device)
        # measured at N = 2 (baby x2, profiles/): barriers as separate launches 0.165 ms per propagation, inside the
        # kernels 0.21-0.25 ms (the handshake at system scope inside a kernel that also holds SMs costs more than the two
        # launches it saves) -> launches are the default, MMREC_PEER_SYNC=kernel selects the fused form
        self.sync_in_kernel = os.environ.get("MMREC_PEER_SYNC", "launch") == "kernel"

    @staticmethod
    def words(n_users, d, n_layers, n_local, k):
        n = n_users * d
        w = 2 * n_layers * n + n_local * d + ((n_local * d) & 1)
        w += n_users * k + ((n_users * k) & 1) + 2 * n_users * k
        return w + 2 * 16                                            # + the barrier flags (2 * world ints, world <= 16)

    def topk_lists(self, row0, nrows):
        """(values, indices) views of this rank's list region for user rows [row0, row0 + nrows), and the peers' raw
        addresses of the same regions (rank order)."""
        k = self.k
        v = self.buf[self.val_off + row0 * k: self.val_off + (row0 + nrows) * k].view(nrows, k)
        i = self.buf[self.idx_off + 2 * row0 * k: self.idx_off + 2 * (row0 + nrows) * k].view(torch.int64).view(nrows, k)
        vp = [int(p) + 4 * (self.val_off + row0 * k) for p in self.hdl.buffer_ptrs]
        ip = [int(p) + 4 * (self.idx_off + 2 * row0 * k) for p in self.hdl.buffer_ptrs]
        return v, i, vp, ip

    @staticmethod
    def create(n_users, d, n_layers, n_local, device, group=None, k=50):
        try:
            import torch.distributed._symmetric_memory as symm
            grp = group or dist.group.WORLD
            if (n_users * d) % 4:
                return None
            buf = symm.empty(PeerExchange.words(n_users, d, n_layers, n_local, k), dtype=torch.float32, device=device)
            hdl = symm.rendezvous(buf, grp)
            buf.zero_()
            px = PeerExchange(hdl, buf, n_users, d, n_layers, n_local, dist.get_rank(grp), dist.get_world_size(grp), n_users, k)
            px.barrier()
            torch.cuda.synchronize(device)
            return px
        except Exception:                                            # noqa: BLE001
            return None

    def barrier(self):
        """Device-side barrier of all ranks on the current stream.  Successive barriers rotate over the signal channels
        (every rank issues them in the same order, so a channel is never shared by two barriers in flight)."""
        self.hdl.barrier(channel=self._chan)
        self._chan = (self._chan + 1) % 8


def propagate_mean_sharded_p2p(a_ui, a_iu, user_emb, item_emb_local, n_layers, px: PeerExchange, mm_local=None):
    """`propagate_mean_sharded` with the all-reduce replaced by this library's kernel over peer memory, in the
    reduce-scatter + all-gather form: the user-side SpMM writes its partial into the symmetric buffer, the item-side SpMM
    runs meanwhile on a second stream; barrier; `mmrec_peer_reduce_push_f32` sums THIS rank's 1/world slice of all
    partials (rank order) and stores it into every rank's reduced table; barrier.  Per layer and rank (world-1)/world of
    [U, d] is read and as much written over NVLink.  The running layer sum of the users lives sliced (each rank its
    slice), the final layer stores (acc + sum) / (L + 1) -- the propagated user table -- instead of the sum.

    `mm_local` (FREEDOM's item-item layer, `src/models/freedom.py:166-167,178`): CSR of this rank's rows of mm_adj with
    rank-major columns (`ItemShard.mm_csr`); the layer-0 item embeddings are gathered from the peers that own them
    (`mmrec_peer_gather_f32`) and `i_g += mm_adj @ E_I`.  Returns (u_g [U, d] -- a view of the exchange buffer, valid
    until the next call --, i_g [I_local, d])."""
    from . import ops
    U, d = user_emb.shape
    dev = user_emb.device
    eu, ei = user_emb, item_emb_local
    acc_i = item_emb_local.clone()
    main = torch.cuda.current_stream()
    side = _side_stream(dev)
    hh = None
    _mark("start")
    if mm_local is not None:
        # The item-item term needs layer-0 rows only, so it runs on the second stream from the start, underneath the UI
        # layers: publish my item rows, barrier, gather the peers' rows straight from their memory, hh = mm_adj @ E_I.
        px.items.copy_(item_emb_local)
        side.wait_stream(main)
        with torch.cuda.stream(side):
            px.barrier()
            ei_all = torch.empty(px.world * px.n_local, d, dtype=torch.float32, device=dev)
            ops.peer_gather(px.item_ptrs, px.n_local * d, ei_all)
            hh = torch.empty(px.n_local, d, dtype=torch.float32, device=dev)
            ops.spmm_raw(mm_local, ei_all, Y=hh)
    ue_flat = user_emb.reshape(-1)
    for l in range(1, n_layers + 1):
        last = l == n_layers
        div = float(n_layers + 1) if last else 1.0
        # the two SpMMs of a layer read only layer l-1: side by side on two streams (fork / join with events, so the pair
        # is also a valid CUDA-graph capture)
        side.wait_stream(main)
        with torch.cuda.stream(side):
            ei_next, acc_i = _cuda_spmm(a_iu, eu, acc_in=acc_i, acc_div=div, want_y=not last)
        ops.spmm_raw(a_ui, ei, Y=px.parts[l - 1])                    # R_g E_Ig -> peer-visible partial of layer l
        _mark(f"L{l} user-side spmm")
        acc_in = ue_flat[px.lo:px.hi] if l == 1 else px.acc
        if px.sync_in_kernel:
            # one launch: wait for every rank's partial, reduce my slice, store it to every rank, wait for every rank's stores
            ops.peer_exchange(px.part_ptrs[l - 1], px.gath_ptrs[l - 1], px.flag_ptrs, px.state, U * d, px.rank, acc_in=acc_in,
                              acc_out=px.acc, acc_div=div, final_layer=last)
        else:
            px.barrier()                                             # every rank's partial of layer l is complete
            _mark(f"L{l} barrier A")
            ops.peer_reduce_push(px.part_ptrs[l - 1], px.gath_ptrs[l - 1], U * d, px.rank, acc_in=acc_in, acc_out=px.acc, acc_div=div,
                                 final_layer=last)
            _mark(f"L{l} reduce+push")
            px.barrier()                                             # every slice of the reduced table has landed
        _mark(f"L{l} barrier B")
        main.wait_stream(side)
        _mark(f"L{l} join item-side stream")
        eu, ei = px.gath[l - 1], ei_next
    u_g = px.gath[n_layers - 1] if n_layers > 0 else user_emb
    if mm_local is not None:
        main.wait_stream(side)
        acc_i = acc_i + hh                                           # i_g + mm_adj @ E_I  (freedom.py:178)
    _mark("end")
    return u_g, acc_i


_side = {}
_timing = None                                                      # tuning aid: list of (label, event) while MMREC_SHARDED_TIMING is set


def _mark(label):
    if _timing is not None:
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        _timing.append((label, e))


def timed_phases(fn, reps=3):
    """Run `fn` eagerly `reps` times with CUDA events between the phases of `propagate_mean_sharded_p2p`; returns
    [(label, mean microseconds since the previous mark)]."""
    global _timing
    acc = {}
    order = []
    for _ in range(reps):
        _timing = []
        fn()
        torch.cuda.synchronize()
        for (l0, e0), (l1, e1) in zip(_timing[:-1], _timing[1:]):
            if l1 not in acc:
                acc[l1] = 0.0; order.append(l1)
            acc[l1] += e0.elapsed_time(e1) * 1e3 / reps
    _timing = None
    return [(l, acc[l]) for l in order]


def _side_stream(device):
    key = torch.device(device).index
    if key not in _side:
        _side[key] = torch.cuda.Stream(device=device)
    return _side[key]


def merge_rows(B, world, rank):
    """Rows of a B-row batch that rank `rank` merges: a contiguous slice."""
    per = (B + world - 1) // world
    lo = min(per * rank, B)
    return lo, min(lo + per, B) - lo


def score_topk_sharded_p2p(shard: ItemShard, user_e, item_e_local, users, lmask, k, px: PeerExchange, row0, catalog=None):
    """`score_topk_sharded` without a collective: the fused score+top-k kernels write this rank's (value, local item)
    lists straight into peer-mapped memory, one device barrier, then every rank merges ITS slice of the batch rows from
    all ranks' lists (`mmrec_topk_merge_peers`, which also relabels local -> global item ids).  Returns (values, indices,
    first row, rows) of that slice; `lmask` is the output of `local_mask`."""
    from . import ops
    B = users.numel()
    v, i, vp, ip = px.topk_lists(row0, B)
    ops.score_topk(user_e, item_e_local, users, lmask, k, out=(v, i), catalog=catalog)
    lo, cnt = merge_rows(B, shard.world, shard.rank)
    sync = None
    if px.sync_in_kernel:
        sync = (px.flag_ptrs, px.state, px.rank)                    # the merge kernel waits for the peers' lists itself
    else:
        px.barrier()
    mv, mi = ops.topk_merge_peers(vp, ip, B, k, user_e.device, idx_mul=shard.world, idx_add=1, row0=lo, n_rows=cnt, sync=sync)
    return mv, mi, lo, cnt


def local_mask(shard: ItemShard, mask):
    """The entries of a [2, nnz] (batch row, GLOBAL item) mask that fall on this rank's shard, relabelled to local
    item ids.  Data-dependent size: done once per batch by whoever builds the batches, outside the step."""
    if mask is None or mask.numel() == 0:
        return None
    sel = (mask[1] % shard.world) == shard.rank
    return torch.stack([mask[0][sel], mask[1][sel] // shard.world])


def score_topk_sharded(shard: ItemShard, user_e, item_e_local, users, mask, k, score_topk=None, merge=None, group=None,
                       mask_is_local=False):
    """Global top-k over all shards.  `mask` holds GLOBAL item ids ([2, nnz]: batch row, item) unless
    `mask_is_local` (then it is the output of `local_mask`)."""
    from . import ops
    score_topk = score_topk or ops.score_topk
    merge = merge or ops.topk_merge
    world = shard.world
    lm = mask if mask_is_local else local_mask(shard, mask)
    val, idx = score_topk(user_e, item_e_local, users, lm, k)
    idx = idx * world + shard.rank                                   # back to global item ids
    B = val.shape[0]
    # one collective per batch: (value bits, global item id) as an int32 pair (item ids are < 2^31, checked by the shard)
    pair = torch.stack([val.contiguous().view(torch.int32), idx.to(torch.int32)], dim=-1)          # [B, k, 2]
    allp = torch.empty(world, B, k, 2, dtype=torch.int32, device=val.device)
    dist.all_gather_into_tensor(allp.view(world * B, k * 2), pair.view(B, k * 2), group=group)
    vals = allp[..., 0].contiguous().view(torch.float32)
    idxs = allp[..., 1].to(torch.int64)
    return merge(vals, idxs)


# ------------------------------------------------------------------------------------------------------
# single-GPU comparison of the sharded result (SURVEY.md 8e: the correctness oracle for multi-GPU = the 1-GPU kernels)
# ------------------------------------------------------------------------------------------------------
def parity_vs_single_gpu(wl, shard, u_g, i_g, eval_out, batches, kr, kc, kv, n_layers, k, dev):
    """Every rank recomputes the whole (unsharded) problem with the single-GPU kernels on its own device and compares:
    user table and its item shard (relative error, bar 1e-4), and its slice of every batch's merged top-k (index
    mismatches must be near ties under an fp64 re-score of the single-GPU embeddings).  Returns a dict of plain numbers,
    reduced over ranks (max of errors, sum of counts)."""
    from . import graph, ops
    from .ops import CSR
    U, I = wl.U, wl.I
    adj = graph.build_norm_adj((wl.tr_u, wl.tr_i), U, I, dev)
    ego = torch.from_numpy(np.concatenate([wl.user_emb, wl.item_emb])).to(dev)
    all_emb = ops.propagate_mean(adj, ego, n_layers)
    u_ref, i_ref = all_emb[:U], all_emb[U:]
    if kr is not None:
        mm = CSR.from_coo(torch.from_numpy(kr).to(dev), torch.from_numpy(kc).to(dev), torch.from_numpy(kv).to(dev), I, I)
        i_ref = ops.spmm(mm, ego[U:], base=i_ref)
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()
    u_err = rel(u_g, u_ref)
    i_err = rel(i_g, i_ref[torch.from_numpy(shard.local_items).to(dev)])
    rows = mism = non_tie = 0
    i64 = i_ref.double()
    for (users, mask, _), (mv, mi, lo, cnt) in zip(batches, eval_out):
        if cnt == 0:
            continue
        us = users[lo:lo + cnt]
        sel = (mask[0] >= lo) & (mask[0] < lo + cnt)
        m = torch.stack([mask[0][sel] - lo, mask[1][sel]])
        _, ref_idx = ops.score_topk(u_ref, i_ref, us, m, k)
        rows += cnt
        bad = (ref_idx != mi).any(dim=1).nonzero().flatten()
        mism += int(bad.numel())
        if bad.numel():                                             # near-tie rule on an fp64 re-score of the reference embeddings
            s = u_ref[us[bad]].double() @ i64.t()
            scale = s.abs().max().item()
            got, want = s.gather(1, mi[bad]), s.gather(1, ref_idx[bad])
            non_tie += int(((got - want).abs().max(dim=1).values > 4e-6 * scale).sum().item())
    t = torch.tensor([u_err, i_err], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    c = torch.tensor([rows, mism, non_tie], device=dev, dtype=torch.float64)
    dist.all_reduce(c, op=dist.ReduceOp.SUM)
    u_err, i_err = t.tolist()
    rows, mism, non_tie = [int(x) for x in c.tolist()]
    return {"vs": "single-GPU kernels on the unsharded problem (every rank, own device)", "user_emb_rel_err": u_err,
            "item_emb_rel_err": i_err, "topk_rows_checked": rows, "topk_rows_with_index_mismatch": mism,
            "topk_rows_beyond_near_tie": non_tie, "ok": bool(u_err < 1e-4 and i_err < 1e-4 and non_tie == 0 and rows > 0)}


# ------------------------------------------------------------------------------------------------------
# bench driver for N > 1 (weak scaling: every rank keeps 7,000 items and ~160k edges as N grows)
# ------------------------------------------------------------------------------------------------------
def bench_sharded(args, rank, world, dev, Workload, peaks, ClockSampler):
    from . import ops
    TOPK, EVAL_BATCH = 50, 4096
    wl = Workload(args.workload, n_layers=3, items_scale=world)
    U, I, d = wl.U, wl.I, wl.d
    shard = ItemShard(wl.tr_u, wl.tr_i, U, I, rank, world)
    a_ui, a_iu = shard.csrs(dev, d)
    kr, kc, kv = wl.knn_coo()
    mm_local = shard.mm_csr(kr, kc, kv, dev, d)                     # FREEDOM's item-item layer: this rank's rows, rank-major columns
    ue = torch.from_numpy(wl.user_emb).to(dev)
    ie = torch.from_numpy(wl.item_emb[shard.local_items]).to(dev)
    U_eval = min(U, 8 * EVAL_BATCH) if U > 16 * EVAL_BATCH else U    # (very large jobs: a bounded sample of the user batches per step)
    batches = []
    for lo in range(0, U_eval, EVAL_BATCH):
        hi = min(U_eval, lo + EVAL_BATCH)
        m = torch.from_numpy(wl.eval_mask(lo, hi)).to(dev)
        batches.append((torch.arange(lo, hi, device=dev), m, local_mask(shard, m)))
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    edges_local = wl.n_layers * 2 * shard.nnz + mm_local.nnz
    ev = lambda: torch.cuda.Event(enable_timing=True)
    tA = tC = 0.0
    sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0")))
    state = {}

    px = None if (world == 1 or os.environ.get("MMREC_EXCHANGE", "p2p") == "nccl") else PeerExchange.create(U, d, wl.n_layers, shard.n_local, dev, k=TOPK)
    have = torch.tensor([1.0 if px is not None else 0.0], device=dev)
    dist.all_reduce(have, op=dist.ReduceOp.MIN)
    if have.item() == 0.0:
        px = None
    exchange = ("mmrec_peer_reduce_push_f32 (reduce-scatter + all-gather over symmetric memory: each rank sums its 1/N slice of the partials "
                "and stores it to every peer), mmrec_peer_gather_f32 for the item-item layer, mmrec_topk_merge_peers on 1/N of the rows; "
                "no NCCL collective on the data path" if px is not None else "NCCL all-reduce + all-gather")

    def prop(u_in, i_in):
        if px is not None:
            return propagate_mean_sharded_p2p(a_ui, a_iu, u_in, i_in, wl.n_layers, px, mm_local=mm_local)
        u, i = propagate_mean_sharded(a_ui, a_iu, u_in, i_in, wl.n_layers)
        return u, mm_layer_sharded(shard, mm_local, i_in, i)

    def sec_a():
        return prop(ue, ie)

    def score_batch(bi, u_g, i_g, users, lm, cat=None):
        if px is not None:
            return score_topk_sharded_p2p(shard, u_g, i_g, users, lm, TOPK, px, bi * EVAL_BATCH, catalog=cat)
        v, i = score_topk_sharded(shard, u_g, i_g, users, lm, TOPK, mask_is_local=True)
        return v, i, 0, users.numel()

    def sec_c():
        cat = ops.Catalog(state["i"])                               # the shard's item operand: packed once per evaluation
        return [score_batch(bi, state["u"], cat.item_e, users, lm, cat) for bi, (users, _, lm) in enumerate(batches)]

    # ---- parity first: the sharded result against the single-GPU kernels, on every rank (SURVEY.md 8e)
    with torch.no_grad():
        state["u"], state["i"] = sec_a()
        out_c = sec_c()
        torch.cuda.synchronize(); dist.barrier()
        parity = parity_vs_single_gpu(wl, shard, state["u"], state["i"], out_c, batches, kr, kc, kv, wl.n_layers, TOPK, dev)
        del out_c
    torch.cuda.synchronize(); dist.barrier()

    # Both sections (kernels of 5-70 us, barriers / collectives included) are captured once into CUDA graphs and replayed,
    # as in the single-GPU arm; if this torch/NCCL build refuses to capture something the arm runs them eagerly.
    graphs, n_launch, mode = {}, {"a": 0, "c": 0}, "cuda graphs"
    side = torch.cuda.Stream()
    with torch.cuda.stream(side), torch.no_grad():
        for _ in range(2):
            state["u"], state["i"] = sec_a(); sec_c()
        torch.cuda.synchronize(); dist.barrier()
        try:
            for name, fn in (("a", sec_a), ("c", sec_c)):
                l0 = ops.launch_count()
                gph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gph, stream=side):
                    out = fn()
                graphs[name], n_launch[name] = gph, ops.launch_count() - l0
                if name == "a":
                    state["u"], state["i"] = out
            torch.cuda.synchronize()
        except Exception as exc:                                     # noqa: BLE001
            graphs, mode = {}, f"eager ({type(exc).__name__} during graph capture)"
            torch.cuda.synchronize()
    ok = torch.tensor([1.0 if graphs else 0.0], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)                        # all ranks replay, or none
    if ok.item() == 0.0:
        graphs = {}
    launches = 0
    with torch.no_grad():
        for step in range(args.warmup + args.steps):
            if step == 0 and rank == 0:
                sampler.start()
            if step == args.warmup:
                torch.cuda.synchronize(); dist.barrier()
            flush.zero_()
            torch.cuda.synchronize(); dist.barrier()
            e = [ev() for _ in range(4)]
            l0 = ops.launch_count()
            e[0].record()
            if graphs:
                graphs["a"].replay()
            else:
                state["u"], state["i"] = sec_a()
            e[1].record()
            e[2].record()
            if graphs:
                graphs["c"].replay()
            else:
                sec_c()
            e[3].record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                tA += e[0].elapsed_time(e[1]); tC += e[2].elapsed_time(e[3])
                launches += (n_launch["a"] + n_launch["c"]) if graphs else ops.launch_count() - l0
    dist.barrier()
    phases = None
    if os.environ.get("MMREC_SHARDED_TIMING") and px is not None:
        with torch.no_grad():
            phases = timed_phases(lambda: prop(ue, ie))
        dist.barrier()
    # ---- e2e: the same calls with pinned HOST buffers, copies inside the timed region
    ue_h = torch.from_numpy(wl.user_emb).pin_memory()
    ie_h = torch.from_numpy(wl.item_emb[shard.local_items]).pin_memory()
    out_u = torch.empty(U, d).pin_memory(); out_i = torch.empty(shard.n_local, d).pin_memory()
    users_h = [b[0].cpu().pin_memory() for b in batches]
    masks_h = [b[2].cpu().pin_memory() for b in batches]             # this rank's share of the mask
    out_idx = [torch.empty(merge_rows(b[0].numel(), world, rank)[1] if px is not None else b[0].numel(), TOPK, dtype=torch.int64).pin_memory()
               for b in batches]
    eA = eC = 0.0
    with torch.no_grad():
        for step in range(args.warmup + args.steps):
            flush.zero_()
            dist.barrier()
            e = [ev() for _ in range(4)]
            e[0].record()
            ue_d, ie_d = ue_h.to(dev, non_blocking=True), ie_h.to(dev, non_blocking=True)
            u_g, i_g = prop(ue_d, ie_d)
            out_u.copy_(u_g, non_blocking=True); out_i.copy_(i_g, non_blocking=True)
            e[1].record()
            e[2].record()
            cat = ops.Catalog(i_g)
            for bi, (uh, mh, oh) in enumerate(zip(users_h, masks_h, out_idx)):
                res = score_batch(bi, u_g, cat.item_e, uh.to(dev, non_blocking=True), mh.to(dev, non_blocking=True), cat)
                oh.copy_(res[1], non_blocking=True)
            e[3].record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                eA += e[0].elapsed_time(e[1]); eC += e[2].elapsed_time(e[3])
    dist.barrier()
    h2d = (ue_h.numel() + ie_h.numel()) * 4 + sum(u.numel() * 8 + m.numel() * 8 for u, m in zip(users_h, masks_h))
    d2h = (out_u.numel() + out_i.numel()) * 4 + sum(o.numel() * 8 for o in out_idx)
    t = torch.tensor([tA, tC, eA, eC], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)                          # device time of the slowest rank
    e_all = torch.tensor([float(edges_local), float(launches), float(h2d), float(d2h)], device=dev, dtype=torch.float64)
    dist.all_reduce(e_all, op=dist.ReduceOp.SUM)                      # units processed / kernels launched / bytes copied by all ranks
    clocks = sampler.stop() if rank == 0 else None
    if rank == 0:
        K = args.steps
        msA, msC = t[0].item() / K, t[1].item() / K
        edges = e_all[0].item()
        pk = peaks()
        algo_bytes = (wl.n_layers * (a_ui.algorithmic_bytes(d) + a_iu.algorithmic_bytes(d)) + mm_local.algorithmic_bytes(d)) * world
        nvl_bytes = wl.n_layers * 2 * (world - 1) / world * U * d * 4 + (world - 1) * shard.n_local * d * 4   # per rank: slices read + pushed, item rows gathered
        print(json.dumps({
            "metric": f"graph-prop edges/sec (+ full-catalog scored-items/sec in extra) @ d={d}",
            "value": edges / (msA * 1e-3), "unit": "edges/s", "n_gpus": world, "steps": K, "warmup": args.warmup,
            "ms_per_step": msA + msC, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": {"workload": f"FREEDOM synthetic {wl.name} x{world} items: {U} users, {I} items ({I // world} per GPU), "
                                   f"{len(wl.tr_u)} train edges, d={d}, {wl.n_layers} UI layers + 1 mm layer, top-{TOPK} over "
                                   f"{'all' if U_eval == U else U_eval} users, eval batch {EVAL_BATCH}",
                       "l2": "flushed (512 MiB write) before every step",
                       "parallelism": f"item-sharded x{world}: per layer reduce-scatter + all-gather of the user table, item rows gathered once "
                                      f"for the item-item layer, per-user top-k merge on 1/{world} of the rows per rank",
                       "launch": mode, "user_exchange": exchange},
            "parity": parity,
            "extra": {"prop_ms": msA, "score_topk_ms": msC, "scored_items_per_sec": U_eval * I / (msC * 1e-3), "eval_users_per_step": U_eval,
                      "nvlink_bytes_per_rank_per_step_prop": nvl_bytes,
                      "limiting_collective": "per-layer user-table exchange (2 device barriers + (N-1)/N of [U, d] read and written per rank)",
                      "phases_us_rank0_eager": phases},
            "roofline": {"kernel": "spmm_vec_kernel<64> (per rank: 2 per UI layer + 1 item-item layer)", "bound": "hbm",
                         "achieved": algo_bytes / (msA * 1e-3) / 1e9 / world, "peak": pk["hbm_gbs"], "unit": "GB/s per GPU",
                         "frac": algo_bytes / (msA * 1e-3) / 1e9 / world / pk["hbm_gbs"], "traffic": None, "peak_src": pk["src"],
                         "note": "time includes the per-layer exchange of the user table over NVLink (peer memory), see extra"},
            "gpu_launches": int(e_all[1].item()), "clocks": clocks,
            "e2e": {"value": edges / (t[2].item() / K * 1e-3), "unit": "edges/s", "h2d_bytes_per_step": int(e_all[2].item()),
                    "d2h_bytes_per_step": int(e_all[3].item()), "prop_ms": t[2].item() / K, "score_topk_ms": t[3].item() / K,
                    "scored_items_per_sec": U_eval * I / (t[3].item() / K * 1e-3)},
        }))
    # Shut down in order: the captured graphs hold the barrier / collective work, drop them before the process group.  The
    # daemon timer only fires if the teardown of this torch/NCCL build blocks (rank 0 has printed its line by then).
    import sys
    import threading
    sys.stdout.flush()
    graphs = None
    state.clear()
    torch.cuda.synchronize()
    dist.barrier()
    watchdog = threading.Timer(30.0, lambda: os._exit(0))
    watchdog.daemon = True
    watchdog.start()
    dist.destroy_process_group()
    watchdog.cancel()
