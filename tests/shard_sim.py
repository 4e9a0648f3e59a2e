"""Sequential simulation of the sharded-store semantics with oracle shards -- TEST INFRASTRUCTURE.

S workers, S owners (shards by the ps-lite range rule).  One step:
  [epoch 0] every owner applies the workers' feature counts as separate Update(kFeaCount) calls, rank order;
  every worker pulls the step-start model of its keys, runs Predict / Evaluate / penalty / AUC / CalcGrad with
  the oracle; every owner applies the workers' gradients as separate Update(kGradient) calls in rank order
  (sgd_updater.cc:74-98).  This is what ShardedStore, PeerShardedStore and the fused dfb_shard_* path must equal.
"""
import numpy as np
import torch

from oracle import oracle as O
from oracle_backend import OracleBackend


def key_owner_np(keys, S):
    keys = np.asarray(keys, dtype=np.uint64)
    width = np.uint64(0xFFFFFFFFFFFFFFFF // S)
    return np.minimum(keys // width, np.uint64(S - 1)).astype(np.int64)


GOLDEN = np.uint64(0x9E3779B97F4A7C15)
HOT_SHARED = np.uint64(7 * 0x9E3779B97F4A7C15 % 2**64)     # raw_batch(hot=True): in every 3rd row of every worker, every step


def hot_own(rank):
    """raw_batch(hot=True): the id in every other row of worker `rank`'s batches"""
    return np.uint64((1000 + rank) * 0x9E3779B97F4A7C15 % 2**64)


def raw_batch(rank, step, valued, B=96, ids=500, max_nnz=24, mixed=False, hot=False, seed=0):
    """a raw (un-localized) CSR<u64> minibatch; ids spread over the whole reversed key space.
    Default: small, rows of 0..max_nnz-1 nonzeros.  mixed: row lengths as the kernels' loops see them -- empty rows,
    1..31 nonzeros (one 32-nonzero chunk), 33..200 (several), and three rows of 1024..1500.  hot: hot_own(rank) in
    every other row and HOT_SHARED in every third (B >= ~800 puts both over the owner's hot_split of 256)."""
    rng = np.random.default_rng(100 * rank + step + 7919 * seed)
    if mixed:
        kind = rng.choice(3, B, p=[0.1, 0.6, 0.3])
        nnzr = np.select([kind == 0, kind == 1], [0, rng.integers(1, 32, B)], rng.integers(33, 201, B))
        nnzr[rng.choice(B, 3, replace=False)] = rng.integers(1024, 1501, 3)
    else:
        nnzr = rng.integers(0, max_nnz, B)
    if hot:
        nnzr[::2] = np.maximum(nnzr[::2], 1)
        nnzr[::3] = np.maximum(nnzr[::3], 2)
    off = np.concatenate([[0], np.cumsum(nnzr)]).astype(np.uint64)
    n = int(off[-1])
    idx = rng.integers(0, ids, n).astype(np.uint64) * GOLDEN
    if hot:
        idx[off[:-1][::2].astype(np.int64)] = hot_own(rank)
        idx[off[:-1][::3].astype(np.int64) + 1] = HOT_SHARED
    val = rng.random(n).astype(np.float32) if valued else None
    lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, idx, val, lab


def localized(raw):
    off, idx, val, lab = raw
    lidx, keys, cnt = O.localize(off, idx)
    return dict(nrows=len(lab), nnz=len(idx), U=len(keys), off=torch.from_numpy(off.view(np.int64).copy()),
                lab=torch.from_numpy(lab), lidx=torch.from_numpy(lidx.view(np.int32).copy()),
                keys=torch.from_numpy(keys.view(np.int64).copy()), cnt=torch.from_numpy(cnt),
                val=torch.from_numpy(val) if val is not None else None)


def simulate(S, steps, kw, batch_fn, cnt_steps=2, train_fn=None):
    """batch_fn(rank, step) -> raw batch.  Returns (shards, workers, per-step per-worker progress snapshots)"""
    shards = [OracleBackend(**kw) for _ in range(S)]
    workers = [OracleBackend(**kw) for _ in range(S)]      # fm_step + progress only
    per_step = []
    for step in range(steps):
        is_train = True if train_fn is None else train_fn(step)
        batches = [localized(batch_fn(r, step)) for r in range(S)]
        owners = [key_owner_np(b["keys"].numpy().view(np.uint64), S) for b in batches]
        if step < cnt_steps:
            for s in range(S):
                for r in range(S):
                    m = owners[r] == s
                    shards[s].feacnt(batches[r]["keys"][m], batches[r]["cnt"][m])
        pulled, grads = [], []
        before = [w.progress.copy() for w in workers]
        for r in range(S):
            b = batches[r]
            U, ks = b["U"], shards[0].ks
            w, hasv, V = torch.zeros(U), torch.zeros(U, dtype=torch.int32), torch.zeros(U, ks)
            for s in range(S):
                m = np.nonzero(owners[r] == s)[0]
                ws, hs, Vs = torch.zeros(len(m)), torch.zeros(len(m), dtype=torch.int32), torch.zeros(len(m), ks)
                shards[s].pull_rows(b["keys"][m], ws, hs, Vs)
                w[m], hasv[m], V[m] = ws, hs, Vs
            pulled.append((w, hasv, V))
            gw, gV = torch.zeros(U), torch.zeros(U, ks)
            workers[r].fm_step(b, w, hasv, V, is_train, gw, gV)
            grads.append((gw, gV))
        per_step.append([workers[r].progress - before[r] for r in range(S)])
        if not is_train:
            continue
        for s in range(S):
            for r in range(S):
                m = np.nonzero(owners[r] == s)[0]
                shards[s].push_rows(batches[r]["keys"][m], grads[r][0][m], pulled[r][1][m], grads[r][1][m])
    return shards, workers, per_step


def all_keys(S, steps, batch_fn):
    ks = []
    for r in range(S):
        for st in range(steps):
            off, idx, _, _ = batch_fn(r, st)
            ks.append(O.localize(off, idx)[1])
    return np.unique(np.concatenate(ks))


# ---------------------------------------------------------------------------------------------------------------------
# the CUDA side: S fused-sharded engines in one process, compared with simulate()
# ---------------------------------------------------------------------------------------------------------------------
STATE_TOL = dict(rtol=1e-3, atol=1e-5)


def check_shard(E, shard, keys, what, tol=STATE_TOL):
    """owner E's entries of keys == the simulated shard's: feature counts, has-V exact; w/sqrt_g/z, V, cg within tol"""
    from util import assert_close, oracle_state
    scal, hasv, V, cg = E.read_entries(keys)
    oscal, ohasv, oV, ocg = oracle_state(shard.M, keys)
    assert np.array_equal(hasv, ohasv), what
    assert np.array_equal(scal[:, 0], oscal[:, 0]), what                     # feature counts: exact
    assert_close(scal[:, 1:], oscal[:, 1:], what=f"{what} w/sqrt_g/z", **tol)
    assert_close(V, oV, what=f"{what} V", **tol)
    assert_close(cg, ocg, what=f"{what} cg", **tol)
    assert E.table_stats()["n_keys"] == shard.M.size(), what


def check_progress(pr, ref, what, pen_rtol=1e-4):
    # ref = [loss, penalty, auc, nnz_w, nrows]
    assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0]) + 1e-4, (what, "loss", pr.loss, ref[0])
    assert abs(pr.penalty - ref[1]) <= pen_rtol * abs(ref[1]) + 1e-5, (what, "penalty", pr.penalty, ref[1])
    # AUC * n: predictions that are tied in exact arithmetic (rows whose only active feature is the same) are
    # ordered by rounding; each flipped pair moves AUC * n by n / (n_pos * n_neg) <= ~0.05 at these sizes
    if ref[4] > 0:     # (the reference never evaluates an empty batch; a worker without one contributes nothing)
        assert abs(pr.auc - ref[2]) <= 1e-4 * abs(ref[2]) + 0.3, (what, pr.auc, ref[2])
    assert pr.nrows == ref[4], (what, pr.nrows, ref[4])


def make_local(S, kw, devices=None, engine_kw=None, **shard_kw):
    """S engines of this process (on one GPU unless devices says otherwise), connected as one sharded store"""
    from difacto_b200 import capi
    from difacto_b200.sharded import FusedShardedStore
    ekw = dict(table_capacity=1 << 14, shard_timeout_ms=8000)
    ekw.update(engine_kw or {})
    engines = [capi.Engine(device=devices[r] if devices else 0, **ekw, **kw) for r in range(S)]
    shard_kw.setdefault("max_rows", 128)
    shard_kw.setdefault("max_nnz", 4096)
    FusedShardedStore.connect_local(engines, **shard_kw)
    return engines


def enqueue_local(engines, batches, push_cnt, is_train):
    """one step of every rank: batches[r] = (off, idx, val, lab).  One host thread, several engines on one device:
    the five enqueue phases are interleaved (see difacto_b200.h)"""
    for E, (off, idx, val, lab) in zip(engines, batches):
        E.shard_begin_async(len(lab), off, idx, val, lab, push_cnt=push_cnt, is_train=is_train)
    for phase in range(5):
        for E in engines:
            E.shard_phase(phase)


def run_local(S, kw, steps, fn, train_fn=None, devices=None, engine_kw=None, cnt_steps=2, engines=None, **shard_kw):
    """steps of S local ranks on fn(rank, step); returns the engines and every rank's per-step Progress"""
    if engines is None:
        engines = make_local(S, kw, devices, engine_kw, **shard_kw)
    prog = [[] for _ in range(S)]
    for step in range(steps):
        is_train = True if train_fn is None else train_fn(step)
        enqueue_local(engines, [fn(r, step) for r in range(S)], step < cnt_steps, is_train)
        for r in range(S):
            prog[r].append(engines[r].wait_step())
    return engines, prog


def check_vs_simulation(engines, prog, kw, steps, fn, what, train_fn=None, cnt_steps=2, pen_rtol=1e-4,
                        state_tol=STATE_TOL):
    """every rank's Progress and every owner's entries == simulate(); no key on a shard that does not own it.
    pen_rtol: see check_progress, state_tol: see check_shard.  Returns (keys, owner of each key, the simulated shards)"""
    S = len(engines)
    shards, _, per_step = simulate(S, steps, kw, fn, cnt_steps=cnt_steps, train_fn=train_fn)
    for step in range(steps):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"{what} step {step} worker {r}", pen_rtol)
    keys = all_keys(S, steps, fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        check_shard(engines[s], shards[s], keys[own == s], f"{what} shard {s}", state_tol)
        if S > 1:
            _, hasv, _, _ = engines[s].read_entries(keys[own != s])
            assert np.all(hasv == -1), f"{what}: keys of other owners on shard {s}"
    return keys, own, shards
