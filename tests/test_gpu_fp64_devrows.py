"""The device-row store against the float64 one-step reference (fp64_step.py): the pull-compute-push protocol of
ShardedStore / PeerShardedStore (difacto_b200/sharded.py) driven through its C-ABI calls, every rank on one GPU.

A. One worker engine and S owner engines, step by step: dfb_dev_feacnt per owner segment (count push), dfb_dev_pull_rows
   (or dfb_dev_pull_rows_peer into the worker's buffer), dfb_dev_fm_step (or dfb_dev_fm_step_peer, nseg = S, with plain
   device buffers as the owners' receive buffers), dfb_dev_push_rows per owner.  The pre- and post-step state is the
   owners' entries merged in key order; each owner draws its own InitV stream (Reference(streams=...)).  Held: the
   pulled w, has_V pattern and V rows bit for bit, every key within its bound, loss and penalty, every owner's rng
   state and table growth exactly, keys outside the batch unchanged bit for bit.  The worker's forward is k_fm_fast<K, 2>
   (+ k_fm_long) and its gradient rows k_bwd_update<K, ., APPLY = false> at the exact widths; k_fm_generic's atomic
   emission + k_grad_finalize_dense elsewhere; the owner applies pushed rows with k_bwd_update<K, false, true, SRC = 1>
   at the exact widths and k_update_dense_generic elsewhere.  Cases: V_dim 0 .. 257, binary and valued, count push on
   and off, validation steps, an id in 400 rows (the worker reduces it with the whole warp: no pre-reduction), rows at
   and above long_row_nnz, S = 1, 2, 3, 8, every first_seg at S = 3, keys at the ownership boundaries, an owner without
   keys, fewer than 32 keys, 64 keys with first_seg at an empty trailing segment (rot = the padded key count), the
   benchmark's batch at S = 4, and every applicable mutant of the reference rejecting a warm, valued peer step.
   The receive buffers sit between guard rows of NaN: a row stored at a wrong offset is reported, not written elsewhere.
B. S workers x S owners through ShardedStore and PeerShardedStore themselves, one thread per rank: torch.distributed
   is replaced by a thread-level stand-in, and peer_open by the pointers peer_alloc returned (CUDA IPC cannot open a
   handle of its own process).  The two stores agree bit for bit, both agree with shard_sim.simulate, and at S = 1 with
   the fused raw step.
C. Refusals of dfb_dev_fm_step_peer change nothing.
Each case of A prints its largest error-to-bound ratio and its count of ambiguous keys."""
import ctypes
import threading
import time

import numpy as np
import pytest

import bench
import fp64_step as F
import shard_sim
import test_gpu_fp64_paths as P
import test_gpu_fp64_step as S
import test_gpu_lookup_free_step as lf
from oracle import oracle as O
from test_gpu_fused_shard_shapes import LOOSE, boundary_keys

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")
sharded = pytest.importorskip("difacto_b200.sharded")

U64 = np.uint64
EXACT = P.EXACT


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.view(dtype)).cuda()


class DevRows(P.PathRun):
    """one worker engine and S owner engines, on one GPU; the steps of the device-row store, held to the reference.

    peer: the peer calls (exact widths only); first_seg: the worker's first segment (None: 0 for the plain store, as
    the store passes its rank).  order and penalty per launch (engine.cu dev_fm_step_impl): the worker's training step
    at the exact widths is k_fm_fast<K, 2> and k_bwd_update (APPLY = false, its own penalty); every other training step
    k_fm_generic with atomic emission and k_penalty; validation steps k_fm_fast<K, 0> up to 128 and k_penalty"""

    def __init__(self, hp, n_owners, caps, peer=False, engine=lf.ENGINE, amb_frac=F.AMB_FRAC):
        k = hp["V_dim"]
        W = capi.Engine(table_capacity=1024, **engine, **hp)
        S.Run.__init__(self, W, hp, hot_chunk=1 << 30, amb_frac=amb_frac)
        self.owners = [capi.Engine(table_capacity=c, V_capacity=c, **engine, **hp) for c in caps]
        self.S, self.k, self.ks, self.peer = n_owners, k, W.row_stride(), peer
        sms = P.num_sms()
        exact = k in EXACT
        self.order = {"train": "sorted" if exact else "generic", "val": "sorted" if k <= 128 else "generic"}
        self.pen = {"train": F.pen_partial_bwd_worker(sms) if exact else F.pen_partial_warp_per_key(sms),
                    "val": F.pen_partial_warp_per_key(sms)}

    def close(self):
        for E in [self.E] + self.owners:
            E.close()

    def read(self, keys):
        """the owners' entries of keys (any order), each from its owner"""
        own = sharded.key_owner_np(keys, self.S)
        n, k = len(keys), self.k
        out = [np.zeros((n, 4), np.float32), np.zeros(n, np.int32), np.zeros((n, k), np.float32),
               np.zeros((n, k), np.float32)]
        for s in range(self.S):
            m = own == s
            if m.any():
                for o, part in zip(out, self.owners[s].read_entries(keys[m])):
                    o[m] = part
        return tuple(out)

    def step(self, b, push=False, train=True, first_seg=None, mutants=()):
        W, Sn, k, ks = self.E, self.S, self.k, self.ks
        o, l, i, v = b
        keys, lidx, cnt = F.batch_keys(i)
        Uk = len(keys)
        bounds = [int(x) for x in sharded.shard_bounds_np(keys, Sn)]
        seg = list(zip(bounds[:-1], bounds[1:]))
        pre = self.read(keys)
        out = self.outside(keys)
        out_pre = self.read(out)
        seeds = [E.rng_state() for E in self.owners]
        st0 = [E.table_stats() for E in self.owners]
        d_keys, d_cnt = dev(keys.view(np.int64)), dev(cnt.astype(np.float32))
        d_off, d_lidx, d_lab = dev(o.view(np.int64)), dev(lidx.astype(np.uint32).view(np.int32)), dev(l)
        d_val = dev(v) if v is not None else None
        W.read_progress()                                               # Progress of this step only
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if push:
            for (a, c), E in zip(seg, self.owners):
                if c > a:
                    E.dev_feacnt(d_keys[a:c], c - a, d_cnt[a:c])
        w = torch.full((max(Uk, 1),), float("nan"), device="cuda")
        hasv = torch.zeros(max(Uk, 1), dtype=torch.int32, device="cuda")
        V = torch.zeros((max(Uk, 1), max(ks, 1)), device="cuda")
        hasv_own = [torch.zeros(max(c - a, 1), dtype=torch.int32, device="cuda") for a, c in seg]
        torch.cuda.synchronize()          # torch's fills and copies are on its stream, the engines' kernels on theirs
        for (a, c), E, ho in zip(seg, self.owners, hasv_own):
            if c == a:
                continue
            if self.peer:
                E.dev_pull_rows_peer(d_keys[a:c], c - a, w[a:].data_ptr(), hasv[a:].data_ptr(), V[a:].data_ptr(), ho)
            else:
                E.dev_pull_rows(d_keys[a:c], c - a, w[a:], hasv[a:], V[a:])
        torch.cuda.synchronize()
        self.check_pull(b, keys, pre, seeds, push, train, bounds, w, hasv, V, hasv_own)
        if train and self.peer:
            # each owner's receive buffer between `guard` rows of NaN on both sides
            guard = min(max(Uk, 32), 1 << 20)
            bufs = [(torch.full((c - a + 2 * guard,), float("nan"), device="cuda"),
                     torch.full((c - a + 2 * guard, ks), float("nan"), device="cuda")) for a, c in seg]
            f = 0 if first_seg is None else first_seg
            torch.cuda.synchronize()
            W.dev_fm_step_peer(len(l), len(i), d_off, d_lidx, d_val, d_lab, Uk, w, hasv, V, bounds,
                               [g[guard].data_ptr() for g, _ in bufs], [g[guard].data_ptr() for _, g in bufs],
                               first_seg=f)
            torch.cuda.synchronize()
            grads = []
            for (a, c), (gw_b, gV_b) in zip(seg, bufs):
                for name, t in (("gw", gw_b), ("gV", gV_b)):
                    assert bool(torch.isnan(t[:guard]).all() and torch.isnan(t[guard + c - a:]).all()), \
                        f"{name} rows stored outside owner segment [{a}, {c})"
                grads.append((gw_b[guard:guard + c - a], gV_b[guard:guard + c - a]))
        else:
            gw = torch.full((max(Uk, 1),), float("nan"), device="cuda")
            gV = torch.full((max(Uk, 1), max(ks, 1)), float("nan"), device="cuda")
            torch.cuda.synchronize()
            W.dev_fm_step(len(l), len(i), d_off, d_lidx, d_val, d_lab, Uk, w, hasv, V, train, gw, gV)
            torch.cuda.synchronize()
            grads = [(gw[a:c], gV[a:c]) for a, c in seg]
        if train:
            for (a, c), (gw_s, gV_s) in zip(seg, grads):
                assert not bool(torch.isnan(gw_s).any()), f"gradient w rows of [{a}, {c}) not written"
                if k and c > a:
                    m = hasv[a:c] == 1
                    assert not bool(torch.isnan(gV_s[m][:, :k]).any()), f"gradient V rows of [{a}, {c}) not written"
            for (a, c), E, (gw_s, gV_s), ho in zip(seg, self.owners, grads, hasv_own):
                if c > a:
                    E.dev_push_rows(d_keys[a:c], c - a, gw_s, ho if self.peer else hasv[a:c], gV_s)
        torch.cuda.synchronize()
        t_step = time.perf_counter() - t0
        pr = W.read_progress()
        post = self.read(keys)
        st1 = [E.table_stats() for E in self.owners]
        obs = dict(loss=pr.loss, penalty=pr.penalty, nrows=pr.nrows, rng_after=[E.rng_state() for E in self.owners],
                   n_keys_delta=sum(b_["n_keys"] - a_["n_keys"] for a_, b_ in zip(st0, st1)),
                   n_vrows_delta=sum(b_["n_vrows"] - a_["n_vrows"] for a_, b_ in zip(st0, st1)))
        mode = "train" if train else "val"
        what = f"{'peer' if self.peer else 'plain'} S={Sn} {mode} push={push} first_seg={first_seg}"
        R = self.hold(b, mode, push, pre, post, seeds[0], obs, self.order[mode], self.pen[mode], True, what,
                      mutants, t_step, streams=(bounds, seeds))
        F.assert_unchanged(out_pre, self.read(out), out, what)
        if train:
            self.remember(keys, cnt)
        return R

    def check_pull(self, b, keys, pre, seeds, push, train, bounds, w, hasv, V, hasv_own):
        """what the owners stored into the worker's buffer: the reference's pulled w, V-row pattern and V rows (with the
        count push's InitV rows), bit for bit; the peer pull's owner-side flags equal"""
        Uk, k = len(keys), self.k
        ref = F.Reference(b, self.hp, pre, 0, push, "train" if train else "val", "cuda",
                          streams=(bounds, seeds))
        assert np.array_equal(w[:Uk].cpu().numpy(), pre[0][:, 1]), "pulled w differ from the pre-step state"
        got_hv = hasv[:Uk].cpu().numpy()
        want_hv = np.where(ref.hv_pull, 1, -1)
        assert np.array_equal(got_hv, want_hv), "pulled has_V differ from the reference's V-row pattern"
        if self.peer:
            own = np.concatenate([h[:c - a].cpu().numpy() for h, a, c in zip(hasv_own, bounds[:-1], bounds[1:])])
            assert np.array_equal(own[:Uk], want_hv), "the owners' own has_V flags differ from the pulled ones"
        if k:
            hv = np.nonzero(ref.hv_pull)[0]
            assert np.array_equal(V[:Uk, :k].cpu().numpy()[hv], ref.Vp.cpu().numpy()[hv]), \
                "pulled V rows differ (count-push InitV rows?)"


def mid(rng, pool, valued, hot, B=2000, long_rows=(200, 301)):
    return P.mid_batch(rng, pool, B, valued, hot, long_rows)


def caps_for(batches, n_owners):
    keys = np.unique(np.concatenate([F.batch_keys(b[2])[0] for b in batches]))
    own = sharded.key_owner_np(keys, n_owners)
    return [2 * int((own == s).sum()) + 4096 for s in range(n_owners)]


# ---------------------------------------------------------------------------------------------------------------------
# A. widths, stores, batches
# ---------------------------------------------------------------------------------------------------------------------
WIDTHS = [(0, 2, False), (8, 3, False), (8, 3, True), (10, 2, False), (16, 1, True), (16, 8, False), (32, 2, True),
          (40, 3, False), (64, 2, False), (64, 3, True), (100, 8, False), (128, 2, True), (128, 1, False),
          (129, 3, False), (257, 2, False)]


@pytest.mark.parametrize("V_dim,n_owners,peer", WIDTHS)
def test_device_rows_against_fp64(V_dim, n_owners, peer):
    """two steps with the count push (the second gives count-push InitV rows to keys the first made nonzero), binary
    then valued; a warm valued step without it; a validation step on a batch with unseen ids (the pull inserts them)"""
    rng = np.random.default_rng(4000 + 10 * V_dim + n_owners + peer)
    pool = P.pool_of(rng, 30000)
    hot = pool[5]
    bs = [mid(rng, pool[:20000], False, hot), mid(rng, pool[10000:], True, hot), mid(rng, pool[:20000], True, hot),
          mid(rng, np.concatenate([pool, P.pool_of(rng, 10000) + U64(1)]), True, pool[7])]
    hp = P.wide_hp(V_dim) if V_dim > 128 else dict(V_dim=V_dim, **lf.KW)
    run = DevRows(hp, n_owners, caps_for(bs, n_owners), peer=peer)
    run.step(bs[0], push=True)
    run.step(bs[1], push=True)
    assert V_dim == 0 or run.last_n_push > 0
    run.step(bs[2])
    run.step(bs[3], train=False)
    run.close()


def test_rows_at_the_default_long_row_nnz():
    """long_row_nnz = 1024 (the default): rows of 1024 .. 1100 nonzeros go through k_fm_long on the pulled view"""
    rng = np.random.default_rng(1024)
    pool = P.pool_of(rng, 30000)
    bs = [mid(rng, pool, j == 1, pool[3], long_rows=(1024, 1101)) for j in range(2)]
    hp = dict(V_dim=32, **lf.KW)
    run = DevRows(hp, 2, caps_for(bs, 2), peer=True, engine=dict(hot_split=64))
    run.step(bs[0], push=True)
    run.step(bs[1])
    run.close()


# ---------------------------------------------------------------------------------------------------------------------
# A. segment edges of the peer scatter
# ---------------------------------------------------------------------------------------------------------------------
def with_ids(rng, b, extra):
    """b with the ids `extra` written over its first nonzeros, one per row"""
    o, l, i, v = b
    i = i.copy()
    starts = o[:-1].astype(np.int64)[np.diff(o.astype(np.int64)) > 0]
    i[starts[:len(extra)]] = extra
    return o, l, i, v


@pytest.mark.parametrize("first_seg", [0, 1, 2])
def test_peer_every_first_seg_at_three_owners(first_seg):
    """keys on both sides of every ownership boundary; S = 3, the worker starting at each segment"""
    rng = np.random.default_rng(30 + first_seg)
    pool = P.pool_of(rng, 20000)
    bids = O.reverse_bytes_np(boundary_keys(3))
    bs = [with_ids(rng, mid(rng, pool, j % 2 == 1, pool[3]), bids) for j in range(3)]
    hp = dict(V_dim=16, **lf.KW)
    run = DevRows(hp, 3, caps_for(bs, 3), peer=True)
    run.step(bs[0], push=True, first_seg=first_seg)
    run.step(bs[1], push=True, first_seg=first_seg)
    run.step(bs[2], first_seg=first_seg)
    run.close()


def owned_ids(rng, n, n_owners, keep):
    """n distinct ids whose keys belong to the owners in `keep`"""
    ids = np.unique(rng.integers(0, 1 << 40, 50 * n * n_owners).astype(U64) * lf.GOLDEN)
    ids = ids[np.isin(sharded.key_owner_np(O.reverse_bytes_np(ids), n_owners), keep)]
    return rng.permutation(ids)[:n]


def rows_over(rng, ids, B, valued, lens=(1, 9)):
    """B rows over ids, every id in at least one row"""
    n = rng.integers(*lens, B)
    n[-1] += max(len(ids) - int(n.sum()), 0)
    picks = np.concatenate([ids, ids[rng.integers(0, len(ids), int(n.sum()) - len(ids))]])
    return P.idr.csr(rng, n, rng.permutation(picks), valued)


@pytest.mark.parametrize("case", ["owner_without_keys", "fewer_than_32", "64_keys_empty_trailing", "eight_owners"])
def test_peer_segment_edges(case):
    """an owner that receives no keys (S = 3, the middle one); 20 keys; 64 keys all below the last owner's range with
    first_seg = that empty segment (rot = 64 = the padded key count); S = 8 (the most segments), first_seg = 5"""
    rng = np.random.default_rng(len(case))
    S_, first = {"owner_without_keys": (3, 1), "fewer_than_32": (3, 2), "64_keys_empty_trailing": (4, 3),
                 "eight_owners": (8, 5)}[case]
    if case == "owner_without_keys":
        ids = owned_ids(rng, 3000, S_, [0, 2])
    elif case == "fewer_than_32":
        ids = owned_ids(rng, 20, S_, [0, 1, 2])
    elif case == "64_keys_empty_trailing":
        ids = owned_ids(rng, 64, S_, [0, 1, 2])
    else:
        ids = owned_ids(rng, 5000, S_, list(range(8)))
    B = 300 if len(ids) < 100 else 2000
    bs = [rows_over(rng, ids, B, j % 2 == 1) for j in range(3)]
    for b in bs:
        keys = F.batch_keys(b[2])[0]
        bounds = sharded.shard_bounds_np(keys, S_)
        if case == "owner_without_keys":
            assert bounds[1] == bounds[2]
        if case == "fewer_than_32":
            assert len(keys) == 20
        if case == "64_keys_empty_trailing":
            assert len(keys) == 64 and bounds[S_ - 1] == 64
    hp = dict(V_dim=8 if case != "eight_owners" else 64, **dict(lf.KW, V_threshold=1))
    run = DevRows(hp, S_, caps_for(bs, S_), peer=True)
    run.step(bs[0], push=True, first_seg=first)
    run.step(bs[1], push=True, first_seg=first)
    run.step(bs[2], first_seg=first)
    run.close()


# ---------------------------------------------------------------------------------------------------------------------
# A. the benchmark's batch, and sharpness
# ---------------------------------------------------------------------------------------------------------------------
def test_flagship_peer_four_owners():
    """bench.py's flagship batch (65536 x 100, id_bits = 30, V_dim 64, allV): one worker, four owners, the peer store;
    pass 0 with the count push, then pass 1"""
    args = S.bench_args()
    b = bench.gen_raw_batch(args, 1)
    run = DevRows(bench.hyper(args), 4, caps_for([b], 4), peer=True, engine=dict())
    run.step(b, push=True, first_seg=0)
    run.step(b, first_seg=0)
    print(f"peak device memory {S.peak_gb():.1f} GB")
    run.close()


SHARP = ("drop_hot_occ", "xxp_uses_x", "post_update_V_in_xxp", "swap_tile_neighbour", "no_l2_in_grad_w")


def test_every_mutant_rejects_the_peer_step():
    """a fresh step (InitV by the owners' updates) and a warm valued step with a hot id in 400 rows and l2 > 0, S = 2.
    (hot_chunk_dropped / hot_chunk_twice model the single-GPU step's pre-reduction, which the worker does not have;
    no_clamp needs rows past +-20)"""
    rng = np.random.default_rng(64)
    pool = P.pool_of(rng, 300000)
    hp = dict(V_dim=64, **dict(lf.KW, V_threshold=0, V_init_scale=0.2))
    bs = [lf.big_batch(rng, pool, 20000, True, pool[3]) for _ in range(2)]
    run = DevRows(hp, 2, caps_for(bs, 2), peer=True)
    run.step(bs[0], push=True, first_seg=1, mutants=("adagrad_on_new_initv",))
    run.step(bs[1], first_seg=1, mutants=SHARP)
    run.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["V10", "V129", "nseg0", "nseg9", "bounds_end"])
def test_peer_step_refusals_change_nothing(case):
    V_dim = {"V10": 10, "V129": 129}.get(case, 16)
    rng = np.random.default_rng(7)
    pool = P.pool_of(rng, 5000)
    hp = dict(V_dim=V_dim, **lf.KW)
    E = capi.Engine(table_capacity=1 << 15, **lf.ENGINE, **hp)
    for j in range(2):
        o, l, i, v = mid(rng, pool, j == 1, pool[3], B=500)
        E.train_step_raw(o, i, v, l, push_cnt=True, is_train=True)
    o, l, i, v = mid(rng, pool, True, pool[3], B=500)
    keys, lidx, _ = F.batch_keys(i)
    Uk, ks = len(keys), E.row_stride()
    seen = np.union1d(keys, F.batch_keys(pool)[0])
    w, hasv = torch.zeros(Uk, device="cuda"), torch.zeros(Uk, dtype=torch.int32, device="cuda")
    V = torch.zeros((Uk, ks), device="cuda")
    gw, gV = torch.zeros(Uk, device="cuda"), torch.zeros((Uk, ks), device="cuda")
    d = [dev(o.view(np.int64)), dev(lidx.astype(np.uint32).view(np.int32)), dev(v), dev(l)]
    d_keys = dev(keys.view(np.int64))
    torch.cuda.synchronize()
    E.dev_pull_rows(d_keys, Uk, w, hasv, V)            # (inserts the batch's new keys)
    torch.cuda.synchronize()
    before, seed0, st0 = E.read_entries(seen), E.rng_state(), E.table_stats()
    nseg = {"nseg0": 0, "nseg9": 9}.get(case, 2)
    bounds = [0] + [Uk // 2] * max(nseg - 1, 0) + [Uk] if nseg else [Uk]
    if case == "bounds_end":
        bounds[-1] = Uk - 1
    E.read_progress()
    with pytest.raises(capi.DfbError):
        E.dev_fm_step_peer(len(l), len(i), *d, Uk, w, hasv, V, bounds, [gw.data_ptr()] * nseg,
                           [gV.data_ptr()] * nseg, first_seg=0)
    torch.cuda.synchronize()
    F.assert_unchanged(before, E.read_entries(seen), seen, case)
    assert E.rng_state() == seed0 and E.table_stats() == st0
    assert E.read_progress().nrows == 0
    E.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. S workers x S owners through the store classes, one thread per rank
# ---------------------------------------------------------------------------------------------------------------------
class ThreadGroup:
    """the torch.distributed calls sharded.py makes, between the threads of one process on one GPU.  Every exchange
    first synchronises the caller's current stream (what it sends is complete), and ends once every rank has copied
    what it receives; a rank that does not arrive fails the others' Barrier (timeout) instead of leaving them waiting"""

    def __init__(self, n, timeout=120.0):
        self.n = n
        self.bar = threading.Barrier(n, timeout=timeout)
        self.slots = [None] * n
        self.local = threading.local()

    def is_initialized(self):
        return True

    def get_world_size(self, group=None):
        return self.n

    def get_rank(self, group=None):
        return self.local.rank

    def _exchange(self, obj):
        torch.cuda.current_stream().synchronize()
        self.bar.wait()
        self.slots[self.local.rank] = obj
        self.bar.wait()
        return list(self.slots)

    def _done(self):
        torch.cuda.current_stream().synchronize()
        self.bar.wait()

    def all_to_all_single(self, out, inp, out_splits=None, in_splits=None, group=None):
        n, me = self.n, self.local.rank
        ins = in_splits if in_splits is not None else [inp.shape[0] // n] * n
        got = self._exchange((list(ins), inp))
        pos = 0
        for src in range(n):
            splits, t = got[src]
            a = sum(splits[:me])
            m = splits[me]
            assert out_splits is None or out_splits[src] == m, "all_to_all_single: split sizes disagree"
            out[pos:pos + m].copy_(t[a:a + m])
            pos += m
        assert pos == out.shape[0], "all_to_all_single: output size disagrees"
        self._done()

    def all_gather_into_tensor(self, out, inp, group=None):
        got = self._exchange(inp)
        torch.cat(got, out=out)
        self._done()

    def all_gather_object(self, lst, obj, group=None):
        lst[:] = self._exchange(obj)
        self._done()

    def all_reduce(self, t, op=None, group=None):
        got = self._exchange(t.clone())
        t.copy_(torch.stack(got).sum(0))
        self._done()

    def barrier(self, group=None):
        self._done()


@pytest.fixture
def in_process_peers(monkeypatch):
    """peer_open of a handle peer_alloc made in this process: the pointer peer_alloc returned.  Frees them after"""
    made = {}

    def alloc(E, nbytes, _orig=capi.Engine.peer_alloc):
        ptr, h = _orig(E, nbytes)
        made[h] = (E, ptr)
        return ptr, h
    monkeypatch.setattr(capi.Engine, "peer_alloc", alloc)
    monkeypatch.setattr(capi.Engine, "peer_open", lambda E, h: made[h][1])
    yield
    torch.cuda.synchronize()
    for E, ptr in made.values():
        if E.h:
            E.L.dfb_peer_free(E.h, ctypes.c_void_p(ptr))


STORE_KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)


def store_batch(raw, n_owners):
    off, idx, val, lab = raw
    lidx, keys, cnt = O.localize(off, idx)
    return dict(nrows=len(lab), nnz=len(idx), U=len(keys), bounds=sharded.shard_bounds_np(keys, n_owners),
                off=dev(off.view(np.int64)), lab=dev(lab), lidx=dev(lidx.view(np.int32)), keys=dev(keys.view(np.int64)),
                cnt=dev(cnt), val=dev(val) if val is not None else None)


def run_store(kind, n_owners, kw, steps, fn, monkeypatch, cnt_steps=2):
    """every rank's engine after `steps` steps of ShardedStore (kind "plain") or PeerShardedStore ("peer"), one thread
    per rank; and every rank's per-step Progress"""
    grp = ThreadGroup(n_owners)
    monkeypatch.setattr(sharded, "dist", grp)
    engines = [capi.Engine(table_capacity=1 << 15, long_row_nnz=1024, **kw) for _ in range(n_owners)]
    prog = [[] for _ in range(n_owners)]
    stores = [None] * n_owners
    errors = []

    def rank_main(r):
        try:
            grp.local.rank = r
            torch.cuda.set_device(0)
            be = sharded.CudaBackend(engines[r], torch.device("cuda", 0))
            store = sharded.PeerShardedStore(be, max_keys=8192) if kind == "peer" else sharded.ShardedStore(be)
            stores[r] = store
            for st in range(steps):
                with store._ctx():
                    batch = store_batch(fn(r, st), n_owners)
                store.step(batch, True, push_cnt=st < cnt_steps)
                with store._ctx():
                    torch.cuda.current_stream().synchronize()
                prog[r].append(engines[r].read_progress())
        except BaseException as e:         # noqa: BLE001 -- reported by the main thread
            errors.append((r, e))
            grp.bar.abort()
    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(n_owners)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    assert not errors, f"ranks failed: {errors}"
    return engines, prog


def outcome(engines, keys):
    own = sharded.key_owner_np(keys, len(engines))
    return ([E.read_entries(keys[own == s]) for s, E in enumerate(engines)], [E.rng_state() for E in engines],
            [E.table_stats() for E in engines])


@pytest.mark.parametrize("V_dim", [16, 64, 128])
@pytest.mark.parametrize("n_owners", [2, 3])
def test_stores_through_their_classes(V_dim, n_owners, monkeypatch, in_process_peers):
    """valued and binary batches over one id range (most ids in every worker's batch), rows of 1024 .. 1500 nonzeros
    (long_row_nnz = 1024); the peer store == the plain store bit for bit, both == shard_sim.simulate at the tolerances
    test_gpu_fused_shard_shapes.py explains (LOOSE: column lists hundreds of rows long, summed in another order)"""
    kw = dict(STORE_KW, V_dim=V_dim)

    def fn(rank, step):
        return shard_sim.raw_batch(rank, step, (rank + step) % 2 == 0, B=300, ids=3000, mixed=True)
    steps = 3
    keys = shard_sim.all_keys(n_owners, steps, fn)
    runs = {}
    for kind in ("plain", "peer"):
        engines, prog = run_store(kind, n_owners, kw, steps, fn, monkeypatch)
        runs[kind] = (outcome(engines, keys), prog)
        if kind == "plain":
            plain_engines = engines
    (ea, ra, sa), pa = runs["plain"]
    (eb, rb, sb), pb = runs["peer"]
    for s, (x, y) in enumerate(zip(ea, eb)):
        for name, u, w in zip(("scalars", "has_V", "V", "cg"), x, y):
            assert np.array_equal(u, w), f"owner {s}: {name} differ between the plain and the peer store"
    assert ra == rb and sa == sb, "rng state / table stats differ between the plain and the peer store"
    for r in range(n_owners):
        for st in range(steps):
            a, b = pa[r][st], pb[r][st]
            assert a.nrows == b.nrows
            for f in ("loss", "penalty"):
                x, y = getattr(a, f), getattr(b, f)
                assert abs(x - y) <= 1e-6 * abs(x), (f, r, st, x, y)
    shard_sim.check_vs_simulation(plain_engines, pa, kw, steps, fn, f"plain V_dim {V_dim} S {n_owners}", **LOOSE)
    for E in plain_engines:
        E.close()


def test_single_rank_stores_equal_the_fused_raw_step(monkeypatch, in_process_peers):
    kw = dict(STORE_KW, V_dim=64)

    def fn(rank, step):
        return shard_sim.raw_batch(rank, step, step % 2 == 0, B=300, ids=2000, mixed=True, hot=True)
    steps = 4
    keys = shard_sim.all_keys(1, steps, fn)
    E = capi.Engine(table_capacity=1 << 15, long_row_nnz=1024, **kw)
    for st in range(steps):
        off, idx, val, lab = fn(0, st)
        E.train_step_raw(off, idx, val, lab, push_cnt=st < 2, is_train=True)
    want = E.read_entries(keys)
    for kind in ("plain", "peer"):
        engines, _ = run_store(kind, 1, kw, steps, fn, monkeypatch)
        got = engines[0].read_entries(keys)
        assert np.array_equal(got[1], want[1]) and np.array_equal(got[0][:, 0], want[0][:, 0]), kind
        for a, b in zip(got, want):
            np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6, err_msg=kind)
        assert engines[0].rng_state() == E.rng_state(), kind
