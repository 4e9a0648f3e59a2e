"""NVLink-sharded model store: difacto's Store::Pull/Push as NCCL all-to-all of the active rows.

The reference shards keys over ps-lite servers by contiguous ranges of the (reversed) key space
(ps-lite/src/postoffice.cc:127-136) and a worker slices its sorted key list per server
(ps-lite/include/ps/kv_app.h:406-460, DefaultSlicer); difacto's own distributed Store is
`LOG(FATAL) << "not implemented"` (src/store/store.cc:9-11).  Here every rank is both a worker (its
own minibatch) and a server (shard `rank` of the table, one difacto_b200 engine), one process per
GPU, `torch.distributed` for the plumbing:

    counts      all_to_all of the per-owner segment sizes                    (S ints)
    keys        all_to_all_v of the sorted key segments                      (8 B / key)
    [feacnt]    all_to_all_v of the counts; owner applies Update(kFeaCount) per source rank
    Pull        owner gathers {w, has_V, V[ks]} rows (dfb_dev_pull_rows) -> all_to_all_v back
    compute     dfb_dev_fm_step on the pulled dense rows: loss/AUC/penalty + complete gradients
    Push        all_to_all_v of {gw, gV[ks]} -> owner applies FTRL/AdaGrad per source rank, in
                rank order (the reference applies every worker's push as a separate Update in
                arrival order, sgd_updater.cc:74-98; rank order makes it deterministic)

Because the batch's keys are sorted, every owner's keys are ONE contiguous segment, so the
concatenation of what comes back from owners 0..S-1 is already in key order: no permutation pass.

The protocol is backend-agnostic: `CudaBackend` drives the sm_90a engine (the product);
tests/ injects a CPU backend over gloo to check the protocol itself against the oracle.
"""
import contextlib
import os
import time

import numpy as np
import torch
import torch.distributed as dist


def key_owner_np(keys, S):
    """vectorised dfb_key_owner: min(S-1, key // (UINT64_MAX // S)) on reversed keys"""
    keys = np.asarray(keys, dtype=np.uint64)
    width = np.uint64(0xFFFFFFFFFFFFFFFF // S)
    return np.minimum(keys // width, np.uint64(S - 1)).astype(np.int64)


def shard_bounds_np(sorted_keys, S):
    """segment boundaries [S+1] of a sorted key array (DefaultSlicer's lower_bound per range)"""
    keys = np.asarray(sorted_keys, dtype=np.uint64)
    width = 0xFFFFFFFFFFFFFFFF // S
    cuts = np.array([width * i for i in range(1, S)], dtype=np.uint64)
    inner = np.searchsorted(keys, cuts, side="left")
    return np.concatenate([[0], inner, [len(keys)]]).astype(np.int64)


class CudaBackend:
    """one shard = one difacto_b200 engine; all arrays are torch CUDA tensors"""

    def __init__(self, engine, device):
        self.E = engine
        self.device = device
        self.ks = engine.row_stride()
        self.V_dim = engine.V_dim
        self.stream = torch.cuda.ExternalStream(engine.stream(), device=device)

    def empty(self, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def stream_ctx(self):
        """the engine's kernels run on the engine's stream; torch's collectives, barriers and allocations are ordered
        against torch's CURRENT stream: a step must run with the engine's stream current"""
        return torch.cuda.stream(self.stream)

    def feacnt(self, keys, cnt):
        if len(keys):
            self.E.dev_feacnt(keys, len(keys), cnt)

    def pull_rows(self, keys, w, hasv, V):
        if len(keys):
            self.E.dev_pull_rows(keys, len(keys), w, hasv, V)

    def fm_step(self, batch, w, hasv, V, is_train, gw, gV):
        self.E.dev_fm_step(batch["nrows"], batch["nnz"], batch["off"], batch["lidx"], batch.get("val"),
                           batch["lab"], batch["U"], w, hasv, V, is_train, gw, gV)

    def push_rows(self, keys, gw, hasv, gV):
        if len(keys):
            self.E.dev_push_rows(keys, len(keys), gw, hasv, gV)

    def read_progress(self):
        return self.E.read_progress()


class ShardedStore:
    """Store + the worker's minibatch step over S ranks"""

    def __init__(self, backend, group=None):
        self.b = backend
        self.group = group
        self.S = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.ks = backend.ks
        self._buf = {}
        self.timers = None      # set to {} to collect per-phase CUDA-event timings (device tensors only)
        self._marks = []

    def _mark(self, name):
        if self.timers is None:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self._marks.append((name, ev))

    def flush_timers(self):
        """fold the recorded marks into self.timers[name] = [total_ms, count] (synchronises)"""
        if self.timers is None or not self._marks:
            return self.timers
        torch.cuda.synchronize()
        for (n0, e0), (n1, e1) in zip(self._marks[:-1], self._marks[1:]):
            if n1 == "begin":
                continue
            t = self.timers.setdefault(n1, [0.0, 0])
            t[0] += e0.elapsed_time(e1)
            t[1] += 1
        self._marks = []
        return self.timers

    def _get(self, name, n, shape_tail, dtype):
        t = self._buf.get(name)
        need = (n,) + shape_tail
        if t is None or t.shape[0] < n or t.dtype != dtype:
            cap = max(int(n * 1.2) + 16, 16)
            t = self.b.empty((cap,) + shape_tail, dtype)
            self._buf[name] = t
        return t[:n]

    def _a2a(self, out, inp, out_splits, in_splits):
        if self.S == 1:
            out.copy_(inp)
        else:
            dist.all_to_all_single(out, inp, out_splits, in_splits, group=self.group)

    def _ctx(self):
        ctx = getattr(self.b, "stream_ctx", None)
        return ctx() if ctx else contextlib.nullcontext()

    def step(self, batch, is_train=True, push_cnt=False):
        """one minibatch of SGDLearner::IterateData on this rank's batch; collective over ranks.  Runs with the
        backend's stream current (the collectives and the engine's kernels must share one stream order).

        batch: dict(nrows, nnz, U, off, lidx, val|None, lab, keys, cnt|None, bounds[S+1])"""
        with self._ctx():
            return self._step(batch, is_train, push_cnt)

    def _step(self, batch, is_train=True, push_cnt=False):
        S, U, ks = self.S, batch["U"], self.ks
        self._mark("begin")
        bounds = batch["bounds"]
        send = [int(bounds[i + 1] - bounds[i]) for i in range(S)]
        if S == 1:
            recv = list(send)
        else:
            t_send = torch.tensor(send, dtype=torch.int64, device=batch["keys"].device)
            t_recv = torch.empty_like(t_send)
            dist.all_to_all_single(t_recv, t_send, group=self.group)
            recv = [int(x) for x in t_recv.tolist()]
        R = sum(recv)
        seg = np.concatenate([[0], np.cumsum(recv)]).astype(np.int64)
        keys_r = self._get("keys_r", R, (), torch.int64)
        self._a2a(keys_r, batch["keys"], recv, send)
        self._mark("a2a_counts_keys")
        if push_cnt:
            cnt_r = self._get("cnt_r", R, (), torch.float32)
            self._a2a(cnt_r, batch["cnt"], recv, send)
            for src in range(S):    # one Update(kFeaCount) per worker, rank order
                a, b = int(seg[src]), int(seg[src + 1])
                self.b.feacnt(keys_r[a:b], cnt_r[a:b])
        # ---- Pull ----
        w_r = self._get("w_r", R, (), torch.float32)
        hasv_r = self._get("hasv_r", R, (), torch.int32)
        V_r = self._get("V_r", R, (ks,), torch.float32)
        self.b.pull_rows(keys_r, w_r, hasv_r, V_r)
        self._mark("owner_gather")
        w = self._get("w", U, (), torch.float32)
        hasv = self._get("hasv", U, (), torch.int32)
        V = self._get("V", U, (ks,), torch.float32)
        self._a2a(w, w_r, send, recv)
        self._a2a(hasv, hasv_r, send, recv)
        if ks:
            self._a2a(V, V_r, send, recv)
        self._mark("a2a_pull")
        # ---- Predict / Evaluate / CalcGrad ----
        gw = self._get("gw", U, (), torch.float32)
        gV = self._get("gV", U, (ks,), torch.float32)
        self.b.fm_step(batch, w, hasv, V, is_train, gw, gV)
        self._mark("worker_fm")
        if not is_train:
            return
        # ---- Push(kGradient) ----
        gw_r = self._get("gw_r", R, (), torch.float32)
        gV_r = self._get("gV_r", R, (ks,), torch.float32)
        self._a2a(gw_r, gw, recv, send)
        if ks:
            self._a2a(gV_r, gV, recv, send)
        self._mark("a2a_push")
        for src in range(S):        # one Update(kGradient) per worker, rank order
            a, b = int(seg[src]), int(seg[src + 1])
            self.b.push_rows(keys_r[a:b], gw_r[a:b], hasv_r[a:b], gV_r[a:b])
        self._mark("owner_update")


class PeerShardedStore(ShardedStore):
    """Same protocol, but the two row exchanges are fused into the kernels that produce the rows:
    the owner's gather kernel stores {w, has_V, V} straight into the requester's pull buffer and the
    worker's gradient kernel stores {gw, gV} straight into the owner's receive buffer, through
    peer pointers over NVLink (CUDA IPC, one process per GPU).  NCCL carries only the key lists,
    the count matrix and two tiny barriers per step.  Needs the engine's sorted scatter path
    (V_dim in {8,16,32,64,128}); otherwise use ShardedStore."""

    def __init__(self, backend, max_keys, max_recv_keys=None, group=None):
        super().__init__(backend, group)
        E = backend.E
        S, ks = self.S, self.ks
        self.Umax = int(max_keys)
        self.Rmax = int(max_recv_keys if max_recv_keys is not None else max_keys * 1.5 + 1024)
        al = lambda n: (int(n) + 255) // 256 * 256
        # pull buffer (owners store into it): w | hasv | V
        self.off_hasv = al(self.Umax * 4)
        self.off_V = self.off_hasv + al(self.Umax * 4)
        pull_bytes = self.off_V + al(self.Umax * ks * 4)
        # push buffer (workers store into it): gw | gV
        self.off_gV = al(self.Rmax * 4)
        push_bytes = self.off_gV + al(self.Rmax * ks * 4)
        self.pull_ptr, pull_h = E.peer_alloc(pull_bytes)
        self.push_ptr, push_h = E.peer_alloc(push_bytes)
        handles = [None] * S
        if S > 1:
            dist.all_gather_object(handles, (pull_h, push_h), group=self.group)
        self.pull_peer, self.push_peer = [], []
        for r in range(S):
            if r == self.rank:
                self.pull_peer.append(self.pull_ptr)
                self.push_peer.append(self.push_ptr)
            else:
                self.pull_peer.append(E.peer_open(handles[r][0]))
                self.push_peer.append(E.peer_open(handles[r][1]))
        dev = backend.device
        self._tick = torch.zeros(1, device=dev)
        self.hasv_r = torch.empty(self.Rmax, dtype=torch.int32, device=dev)
        if S > 1:
            dist.barrier(group=self.group)

    def _barrier(self):
        if self.S > 1:
            dist.all_reduce(self._tick, group=self.group)

    def _step(self, batch, is_train=True, push_cnt=False):
        S, U, ks, me, E = self.S, batch["U"], self.ks, self.rank, self.b.E
        self._mark("begin")
        bounds = [int(x) for x in batch["bounds"]]
        send = [bounds[i + 1] - bounds[i] for i in range(S)]
        dev = batch["keys"].device
        if S == 1:
            M = [send]
        else:
            t_send = torch.tensor(send, dtype=torch.int64, device=dev)
            t_all = torch.empty(S * S, dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(t_all, t_send, group=self.group)
            M = t_all.view(S, S).tolist()          # M[r][s] = keys rank r sends to owner s
        recv = [int(M[r][me]) for r in range(S)]
        R = sum(recv)
        # every rank sees the whole count matrix, so a buffer overflow anywhere is detected by all ranks
        # in the same step (a local assert on one rank would leave the others waiting in a collective)
        worst_R = max(sum(int(M[r][s]) for r in range(S)) for s in range(S))
        worst_U = max(sum(int(x) for x in M[r]) for r in range(S))
        if worst_R > self.Rmax or worst_U > self.Umax:
            raise RuntimeError(f"peer buffers too small: a rank receives {worst_R} keys (max_recv_keys={self.Rmax}) "
                               f"or sends {worst_U} keys (max_keys={self.Umax}); recreate PeerShardedStore with larger sizes")
        seg = [0]
        for r in range(S):
            seg.append(seg[-1] + recv[r])
        keys_r = self._get("keys_r", R, (), torch.int64)
        self._a2a(keys_r, batch["keys"], recv, send)
        self._mark("a2a_counts_keys")
        if push_cnt:
            cnt_r = self._get("cnt_r", R, (), torch.float32)
            self._a2a(cnt_r, batch["cnt"], recv, send)
            for src in range(S):
                self.b.feacnt(keys_r[seg[src]:seg[src + 1]], cnt_r[seg[src]:seg[src + 1]])
        # ---- Pull: gather + store into the requester's buffer (its key order = owner order) ----
        for ph in range(S):       # ring order: in phase ph every rank stores into a different peer
            src = (me + ph) % S
            n = recv[src]
            if n == 0:
                continue
            off = sum(int(M[src][s]) for s in range(me))     # = requester's bounds[me]
            base = self.pull_peer[src]
            E.dev_pull_rows_peer(keys_r[seg[src]:seg[src + 1]], n, base + off * 4, base + self.off_hasv + off * 4,
                                 base + self.off_V + off * ks * 4, self.hasv_r[seg[src]:seg[src + 1]])
        self._barrier()
        self._mark("pull_gather_store")
        w, hasv, V = self.pull_ptr, self.pull_ptr + self.off_hasv, self.pull_ptr + self.off_V
        # ---- Predict / Evaluate / CalcGrad; gradient rows stored into the owners' buffers ----
        if not is_train:
            gw = self._get("gw", U, (), torch.float32)
            gV = self._get("gV", U, (ks,), torch.float32)
            E.dev_fm_step(batch["nrows"], batch["nnz"], batch["off"], batch["lidx"], batch.get("val"), batch["lab"], U,
                          w, hasv, V, False, gw, gV)
            self._barrier()     # nobody overwrites this pull buffer before every worker is done with it
            self._mark("worker_fm")
            return
        pgw, pgV = [], []
        for s in range(S):
            off = sum(int(M[r][s]) for r in range(me))        # where my segment starts at owner s
            pgw.append(self.push_peer[s] + off * 4)
            pgV.append(self.push_peer[s] + self.off_gV + off * ks * 4)
        E.dev_fm_step_peer(batch["nrows"], batch["nnz"], batch["off"], batch["lidx"], batch.get("val"), batch["lab"], U,
                           w, hasv, V, bounds, pgw, pgV, first_seg=me)
        self._barrier()
        self._mark("worker_fm_store")
        # ---- Push(kGradient): one Update per worker, rank order ----
        for src in range(S):
            n = recv[src]
            if n == 0:
                continue
            a = seg[src]
            E.dev_push_rows(keys_r[a:a + n], n, self.push_ptr + a * 4, self.hasv_r[a:a + n],
                            self.push_ptr + self.off_gV + a * ks * 4)
        self._mark("owner_update")


class FusedShardedStore:
    """The NVLink-sharded store behind the C-ABI (dfb_shard_*, csrc/shard.cu + kernels_shard.cu): the product's
    multi-GPU path.  Unlike ShardedStore / PeerShardedStore above (which move the k-wide rows of the active keys
    to the workers and the gradient rows back, Store::Pull / Push as the reference's ps-lite does), the rows stay
    on their owner: owners compute the partial FM interaction sums of every worker's rows and ship (k+2) floats
    per EXAMPLE; the whole protocol (GPU localizer, slicing, peer stores, step-counter flags) runs on the
    device.  This class only does the plumbing a host has to do once: exchange the mailbox handles (CUDA IPC,
    one process per GPU) through torch.distributed, or wire engines of the same process together.
    Serves every 0 <= V_dim <= 128 with scatter=sorted (dfb_shard_init refuses other configurations: use
    ShardedStore for them)."""

    def __init__(self, engine, max_rows, max_nnz, group=None, seg_keys=0, seg_nnz=0):
        self.E = engine
        self.group = group
        self.S = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.mailbox_bytes = engine.shard_init(self.rank, self.S, int(max_rows), int(max_nnz), int(seg_keys), int(seg_nnz))
        ptr, handle = engine.shard_export()
        if self.S > 1:
            handles = [None] * self.S
            dist.all_gather_object(handles, handle, group=group)
            peers = [ptr if r == self.rank else engine.peer_open(handles[r]) for r in range(self.S)]
            engine.shard_connect(peers)
            dist.barrier(group=group)      # nobody starts storing into a mailbox that is not mapped everywhere yet

    @staticmethod
    def connect_local(engines, max_rows, max_nnz, seg_keys=0, seg_nnz=0):
        """N engines of ONE process (one per GPU, or several on one GPU in tests): rank = position in the list"""
        S = len(engines)
        for r, E in enumerate(engines):
            E.shard_init(r, S, int(max_rows), int(max_nnz), int(seg_keys), int(seg_nnz))
        ptrs = [E.shard_export()[0] for E in engines]
        for E in engines:
            E.shard_connect(ptrs)

    def step_dev(self, nrows, nnz, d_off, d_ids, d_val, d_lab, is_train=True, push_cnt=False):
        """collective: one minibatch of raw CSR<uint64> per rank, arrays already on this rank's GPU"""
        self.E.shard_step_dev(nrows, nnz, d_off, d_ids, d_val, d_lab, push_cnt, is_train)

    def step_host(self, nrows, off, ids, val, lab, is_train=True, push_cnt=False):
        """collective: the same from (pinned) host arrays; H2D is double-buffered against the previous step"""
        self.E.shard_step_async(nrows, off, ids, val, lab, push_cnt, is_train)


# ---------------------------------------------------------------------------------------------
# bench.py --gpus N (N > 1): one process per GPU, launched by torch.distributed.run
# ---------------------------------------------------------------------------------------------
def parity_check(rank, world, local_rank, V_dim, steps=4, B=512, nnz_row=24, ids=3000):
    """Driver-visible multi-GPU parity: a small model is trained (i) by the fused sharded store over all ranks and
    (ii) on rank 0 through the API-faithful plugin calls a maintainer's difacto would make for the same `world`
    workers and `world` servers in bulk-synchronous order -- Store::Pull for every worker (keys sliced per server),
    FMLoss::Predict / CalcGrad, then Store::Push per worker in rank order (dfb_pull / dfb_predict / dfb_calc_grad /
    dfb_push_grad).  The entries of every shard are compared with the corresponding server engine's (both are the
    product's CUDA paths; each is separately checked against the oracle by tests/).  Tolerance: state rel 1e-3 /
    abs 1e-5, flags exact."""
    from difacto_b200 import capi
    kw = dict(V_dim=V_dim, l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)

    def batch(r, st):
        rng = np.random.default_rng(7000 + 100 * r + st)
        off = (np.arange(B + 1, dtype=np.uint64) * np.uint64(nnz_row))
        idx = rng.integers(0, ids, B * nnz_row).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
        return off, idx, lab

    E = capi.Engine(device=local_rank, table_capacity=1 << 16, **kw)
    store = FusedShardedStore(E, max_rows=B, max_nnz=B * nnz_row)
    losses = []
    for st in range(steps):
        off, idx, lab = batch(rank, st)
        store.step_host(B, off, idx, None, lab, is_train=True, push_cnt=st == 0)
        losses.append(E.wait_step().loss)
    # every key any worker touched; each rank reports the entries it owns
    E1 = capi.Engine(device=local_rank, table_capacity=1 << 16, **kw) if rank == 0 else None
    allk = []
    probe = E1 if E1 is not None else E
    for st in range(steps):
        for r in range(world):
            off, idx, _ = batch(r, st)
            allk.append(probe.localize(off, idx, want_cnt=False)[1])
    allk = np.unique(np.concatenate(allk))
    mine = allk[key_owner_np(allk, world) == rank]
    scal, hasv, V, cg = E.read_entries(mine)
    got = [None] * world
    dist.all_gather_object(got, dict(keys=mine, scal=scal, hasv=hasv, V=V, cg=cg, loss=losses))
    E.close()
    if rank != 0:
        return None
    # ---- the same training through the plugin-call API: `world` server engines (all on this GPU), `world` workers ----
    E1.close()
    srv = [capi.Engine(device=local_rank, table_capacity=1 << 16, **kw) for _ in range(world)]   # same seed per server, as above
    F = srv[0]      # any engine serves the stateless calls (localize / predict / calc_grad / evaluate)
    ref_loss = [[0.0] * steps for _ in range(world)]
    for st in range(steps):
        loc = []
        for r in range(world):
            off, idx, lab = batch(r, st)
            lidx, keys, cnt = F.localize(off, idx)
            own = key_owner_np(keys, world)
            loc.append((off, lidx, lab, keys, cnt, [np.nonzero(own == s_)[0] for s_ in range(world)]))
        if st == 0:     # Push(kFeaCount): one Update per worker on every server, rank order (sgd_learner.cc:214-217)
            for s_ in range(world):
                for (_, _, _, keys, cnt, seg) in loc:
                    if len(seg[s_]):
                        srv[s_].push_feacnt(keys[seg[s_]], cnt[seg[s_]])
        pulled = []
        for (_, _, _, keys, _, seg) in loc:     # Store::Pull: the sorted key list sliced per server (kv_app.h:416-429)
            parts = [srv[s_].pull(keys[seg[s_]]) if len(seg[s_]) else (np.zeros(0, np.float32), np.zeros(0, np.int32))
                     for s_ in range(world)]
            pulled.append((np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])))
        grads = []
        for r, (off, lidx, lab, keys, cnt, seg) in enumerate(loc):
            vals, lens = pulled[r]
            w_pos = (np.cumsum(lens) - lens).astype(np.int32)
            V_pos = np.where(lens > 1, w_pos + 1, -1).astype(np.int32)
            pred = F.predict(off, lidx, None, vals, w_pos, V_pos)
            ref_loss[r][st] = F.evaluate(lab, pred)
            grads.append((F.calc_grad(off, lidx, None, lab, vals, pred, w_pos, V_pos), w_pos))
        for s_ in range(world):                  # Store::Push(kGradient): one Update per worker, rank order
            for r, (off, lidx, lab, keys, cnt, seg) in enumerate(loc):
                ix = seg[s_]
                if not len(ix):
                    continue
                lens = pulled[r][1]
                g, w_pos = grads[r]
                lo, hi = int(w_pos[ix[0]]), int(w_pos[ix[-1]] + lens[ix[-1]])
                srv[s_].push_grad(keys[ix], g[lo:hi], lens[ix])
    worst = dict(w=0.0, V=0.0, cg=0.0)
    flag_mismatch, fail, n = 0, 0, 0
    for r in range(world):
        g = got[r]
        rs, rh, rV, rcg = srv[r].read_entries(g["keys"])
        n += len(g["keys"])
        flag_mismatch += int((rh != g["hasv"]).sum()) + int((rs[:, 0] != g["scal"][:, 0]).sum())
        for name, a_, b_ in (("w", g["scal"][:, 1:], rs[:, 1:]), ("V", g["V"], rV), ("cg", g["cg"], rcg)):
            err = np.abs(a_.astype(np.float64) - b_)
            fail += int((err > 1e-5 + 1e-3 * np.abs(b_)).sum())
            worst[name] = max(worst[name], float(err.max()) if err.size else 0.0)
    loss_rel = max(abs(got[r]["loss"][st] - ref_loss[r][st]) / max(abs(ref_loss[r][st]), 1e-9)
                   for r in range(world) for st in range(steps))
    for e_ in srv:
        e_.close()
    return {"checked": True, "what": "fused sharded store over all ranks vs the reference's dataflow through the plugin calls: `world` "
                                     "server engines + `world` workers on rank 0's GPU, Store::Pull (dfb_pull, keys sliced per "
                                     "server) -> dfb_predict / dfb_calc_grad -> Store::Push (dfb_push_grad) per worker in rank "
                                     "order; small shape",
            "shape": {"world": world, "steps": steps, "rows": B, "nnz_per_row": nnz_row, "V_dim": V_dim},
            "entries_compared": n, "flag_or_count_mismatches": flag_mismatch, "values_out_of_tolerance": fail,
            "max_abs_err": worst, "max_rel_loss_err": loss_rel, "tolerance": "abs 1e-5 + rel 1e-3 (state), flags exact",
            "ok": bool(flag_mismatch == 0 and fail == 0 and loss_rel < 1e-4)}


def _measure(args, rank, world, local_rank, benchmod, sampler=None, with_e2e=True):
    """one configuration on `world` GPUs: engines, the NVLink-sharded store, table warm-up, the timed region
    (device-timed, max over ranks), the per-phase timings and (optionally) the end-to-end region"""
    from difacto_b200 import capi
    dev = torch.device("cuda", local_rank)
    kw = benchmod.hyper(args)
    nb = args.working_set
    nnz_row = benchmod.nnz_of(args)
    B, k = args.batch, args.vdim
    N = B * nnz_row
    steps, warm = args.steps, args.warmup

    # per-rank raw batches in pinned host memory (data parallel: every rank has its own file part, sgd_learner.cc:78-89)
    host = benchmod.gen_raw_set(args, nb, 1 + 1000 * rank, torch)
    probe = capi.Engine(device=local_rank, table_capacity=1024, V_dim=k)
    U0 = len(probe.localize(host[0]["off"].numpy().view(np.uint64), host[0]["ids"].numpy().view(np.uint64), want_cnt=False)[1])
    probe.close()
    # this shard sees about (all ranks' keys) / world distinct keys
    cap = int(nb * U0 * 1.15) + 4096
    id_bits = int(np.ceil(np.log2(float(max(args.id_space, 2))))) if args.workload == "synthetic" else 64
    extra = dict(kv.split("=") for kv in args.engine_kw.split(",") if kv)
    E = capi.Engine(device=local_rank, table_capacity=cap, V_capacity=cap, id_bits=min(id_bits, 64), **extra, **kw)
    # criteo-shaped ids carry the feature group in their low bits, so the reversed keys cluster: full-size segments
    seg = 0 if args.workload == "synthetic" else N
    store = FusedShardedStore(E, max_rows=B, max_nnz=N, seg_keys=seg, seg_nnz=seg)
    devb = [dict(off=h["off"].to(dev), lab=h["lab"].to(dev), ids=h["ids"].to(dev)) for h in host]
    torch.cuda.synchronize()

    def step_dev(b, push_cnt=False, train=True):
        d = devb[b]
        store.step_dev(B, N, d["off"], d["ids"], None, d["lab"], is_train=train, push_cnt=push_cnt)

    for p in range(2):      # table warm-up: afterwards every key has reached its steady state
        for b in range(nb):
            step_dev(b, push_cnt=(p == 0))
    E.read_progress()
    for t in range(warm):
        step_dev(t % nb)
    E.sync()
    dist.barrier()
    torch.cuda.synchronize()
    launches0 = E.launch_count()
    if sampler is not None:
        sampler.start()
    wall0 = time.time()
    E.time_mark(0)
    for t in range(steps):
        step_dev((warm + t) % nb)
    E.time_mark(1)
    ms = torch.tensor([E.time_elapsed_ms()], device=dev)
    E.sync()
    dist.barrier()
    wall1 = time.time()
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    launches = E.launch_count() - launches0
    prog = E.read_progress()

    # ---- per-phase CUDA-event timings (separate region): their sum exceeds the step time when phases overlap ----
    E.profile(True)
    for t in range(max(4, steps // 2)):
        step_dev((warm + t) % nb)
    E.sync()
    st = E.profile_read()
    E.profile(False)
    E.read_progress()
    phases = {n: st[n]["ms"] / max(st[n]["count"], 1) for n in ("localize", "shard_slice_scatter", "shard_owner_partials",
                                                                "shard_worker_reduce", "shard_owner_updates")}
    dist.barrier()

    # ---- e2e: raw uint64 CSR from pinned host memory every step + Progress read back ----
    e2e = None
    if with_e2e and not args.no_e2e:
        def run_e2e(nsteps, first):
            loss = 0.0
            for t in range(nsteps):
                h = host[(first + t) % nb]
                store.step_host(B, h["off"], h["ids"], None, h["lab"], is_train=True)
                if t + 1 < nsteps:
                    n_ = host[(first + t + 1) % nb]
                    E.prefetch_raw(B, n_["off"], n_["ids"], None, n_["lab"])
                if t >= 1:
                    loss += E.wait_step().loss      # D2H of step t-1's result while step t runs
            loss += E.wait_step().loss
            return loss

        run_e2e(warm, 0)
        E.sync()
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loss_sum = run_e2e(steps, warm)
        E.sync()
        torch.cuda.synchronize()
        dist.barrier()
        dt = torch.tensor([time.perf_counter() - t0], device=dev)
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        dt = float(dt.item())
        e2e = {"value": steps * B * world / dt, "unit": "examples/s", "h2d_bytes_per_step": int((B + 1) * 8 + N * 8 + B * 4),
               "d2h_bytes_per_step": 64, "ms_per_step": dt / steps * 1e3,
               "api": "dfb_shard_step_async (+ dfb_prefetch_raw) + dfb_wait_step per rank: raw uint64 CSR from pinned host "
                      "memory, Localizer::Compact on the GPU, NVLink-sharded fused step; no NCCL call and no host "
                      "synchronisation inside a step"}
    wall_end = time.time()       # timed region + phase profile + e2e region: the GPU is under load throughout
    st_tab = E.table_stats()
    loss_all = torch.tensor([prog.loss, prog.nrows], device=dev, dtype=torch.float64)
    dist.all_reduce(loss_all)
    E.close()
    return dict(ms=ms, launches=launches, phases=phases, e2e=e2e, st_tab=st_tab, loss_all=loss_all, U0=U0, wall0=wall0, wall1=wall_end,
                B=B, k=k, N=N, nb=nb, steps=steps, warm=warm)


def bench_main(args, rank, world, local_rank, benchmod):
    import json
    from difacto_b200 import capi

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    sampler = benchmod.ClockSampler(local_rank) if rank == 0 else None
    r = _measure(args, rank, world, local_rank, benchmod, sampler=sampler)
    ms, launches, phases, e2e, st_tab, loss_all = r["ms"], r["launches"], r["phases"], r["e2e"], r["st_tab"], r["loss_all"]
    U0, wall0, B, k, N, nb, steps, warm = r["U0"], r["wall0"], r["B"], r["k"], r["N"], r["nb"], r["steps"], r["warm"]
    parity = None
    try:
        parity = parity_check(rank, world, local_rank, k)
    except Exception as e:       # the check must never take the number down with it; a failure is reported as such
        parity = {"checked": False, "error": repr(e)}
    if rank == 0:
        sampler.stop()
        peak, peak_src = benchmod.load_peaks()
        fwd, emit, upd, step_model = benchmod.byte_model(B, N, U0, k)
        # what crosses NVLink per GPU and direction per step: the slices of the batch's structure (per nnz: 8-byte
        # (row, x) payload + 4-byte key index + 4-byte x; every batch is valued on the wire), the partial sums
        # ((k+2) floats per row and owner) one way, p and p*XV ((k+1) floats per row and owner) the other way
        fr = (world - 1) / world
        nvl_out = fr * (U0 * 12 + N * 16) + (world - 1) * B * (k + 2) * 4 + (world - 1) * B * (k + 1) * 4
        rows_model = 2 * U0 * fr * (8 + 4 * (k + 1))       # BASELINE.md section 3: rows of the active keys, pull + push
        nvl = 450.0   # H100 SXM data-sheet NVLink 4 GB/s per direction (not a measured peak)
        upd_ms = phases["shard_owner_updates"]
        line = {
            "metric": benchmod.metric_name(args), "value": steps * B * world / (ms * 1e-3), "unit": "examples/s",
            "n_gpus": world, "steps": steps, "warmup": warm, "ms_per_step": ms / steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": benchmod.workload_config(args, {
                "unique_keys_per_batch": int(U0), "working_set_batches": nb, "table_keys_rank0": int(st_tab["n_keys"]),
                "input": "raw CSR<uint64> per rank, resident in HBM; every step = Localizer::Compact on the GPU + the "
                         "NVLink-sharded fused minibatch",
                "parallelism": f"dp{world} minibatches x table sharded by reversed-key range over {world} GPUs (ps-lite rule); "
                               "owners compute the partial FM interaction sums of every worker's rows (k+2 floats per row "
                               "cross NVLink instead of k floats per key), per-key gradient + FTRL/AdaGrad on the owner; "
                               "peer stores + step-counter flags in peer memory (CUDA IPC), no NCCL in the step"}),
            "roofline": {"bound": "hbm", "kernel": f"k_bwd_update<{k},shard> x {world} workers (owner-side per-key gradient "
                                                   "reduce + FTRL/AdaGrad; the timed phase includes waiting for the workers' p*XV)",
                         "achieved": upd / (upd_ms * 1e-3) / 1e9 if upd_ms > 0 else 0.0, "peak": peak, "unit": "GB/s",
                         "frac": upd / (upd_ms * 1e-3) / 1e9 / peak if upd_ms > 0 else 0.0, "traffic": None,
                         "peak_source": peak_src, "kernel_ms": upd_ms, "algorithmic_bytes": int(upd),
                         "nvlink": {"bytes_out_per_gpu_per_step": int(nvl_out),
                                    "achieved_GBps_over_whole_step": nvl_out / (ms / steps * 1e-3) / 1e9, "peak_GBps": nvl,
                                    "rows_exchange_model_bytes": int(rows_model),
                                    "note": "the step is HBM-bound again: the rows stay on their owner; the row-exchange "
                                            "protocol of round 1 would move rows_exchange_model_bytes per direction"}},
            "cpu_baseline": None, "e2e": e2e, "gpu_launches": int(launches),
            "clocks": sampler.summary(wall0, r["wall1"]), "loss_per_example": float(loss_all[0] / max(loss_all[1], 1)),
            "phases_ms_per_step_rank0": phases, "phases_sum_ms": float(sum(phases.values())), "parity": parity,
        }
    # the Criteo-shaped configurations BASELINE.json names, one short run each on the same ranks.  The headline line
    # is complete at this point: a watchdog prints it and ends the process if a sweep point should ever stall (a
    # rank failing on its own would leave the others waiting in a collective), so the sweep cannot cost the number
    import threading

    def bail():
        if rank == 0:
            line["sweep"] = {"error": "sweep did not finish within its time limit; headline unaffected"}
            print(json.dumps(line), flush=True)
        os._exit(0)

    dog = threading.Timer(150.0, bail)
    dog.daemon = True
    dog.start()
    sweep = None
    if not args.no_sweep and args.workload == "synthetic":
        import argparse
        sweep = {}
        for name, over in (("criteo39_V64_conf", dict(workload="criteo39", vdim=64, hyper="criteo_conf")),
                           ("criteo39_V32_ftrl_l1", dict(workload="criteo39", vdim=32, hyper="ftrl_l1"))):
            a2 = argparse.Namespace(**vars(args))
            a2.steps, a2.warmup, a2.working_set = 6, 3, 4
            for k_, v_ in over.items():
                setattr(a2, k_, v_)
            try:
                r2 = _measure(a2, rank, world, local_rank, benchmod, with_e2e=False)
                sweep[name] = {"value": r2["steps"] * r2["B"] * world / (r2["ms"] * 1e-3), "unit": "examples/s",
                               "ms_per_step": r2["ms"] / r2["steps"], "steps": r2["steps"], "warmup": r2["warm"],
                               "unique_keys_per_batch": int(r2["U0"]), "hyper": benchmod.hyper(a2), "V_dim": a2.vdim,
                               "phases_ms_per_step_rank0": r2["phases"],
                               "loss_per_example": float(r2["loss_all"][0] / max(float(r2["loss_all"][1]), 1.0))}
            except Exception as e:      # a sweep point must not take the headline down
                sweep[name] = {"error": repr(e)}
    dog.cancel()
    if rank == 0:
        line["sweep"] = sweep
        print(json.dumps(line), flush=True)
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
    import sys
    sys.stdout.flush()
    sys.stderr.flush()
    os._exit(0)
