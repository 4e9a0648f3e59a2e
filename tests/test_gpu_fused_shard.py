"""GPU parity tests of the NVLink-sharded store behind the C-ABI (dfb_shard_*): the product's multi-GPU path.

Every test compares the CUDA path with a sequential simulation of the same parameter-server semantics built
on oracle shards (tests/shard_sim.py).  The protocol is exercised
  * with one rank (events only),
  * with 2 and 3 ranks that live in ONE process on ONE GPU (peer pointers are plain device pointers; the step
    counters are polled exactly as between GPUs) -- so the driver's single-GPU test box runs the whole protocol,
  * with one process per GPU over CUDA IPC when 2 GPUs are visible.
Tolerances as in test_gpu_parity.py: model state after T steps rel 1e-3 / abs 1e-5 (fp32, different summation
order over k and over the owners' partials); keys, has-V flags, feature counts bit-exact."""
import ctypes as C
import os
import socket
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import oracle as O  # noqa: E402
from shard_sim import (STATE_TOL, all_keys, check_progress, check_shard, check_vs_simulation, enqueue_local,  # noqa: E402
                       key_owner_np, make_local, raw_batch, run_local, simulate)
from util import assert_close, oracle_state  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(V_dim=16, l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)
STEPS = 6


def batch_fn(rank, step):
    return raw_batch(rank, step, valued=(step % 2 == 0))


@pytest.mark.parametrize("S", [1, 2, 3])
def test_fused_shard_local_ranks_vs_oracle_simulation(S):
    engines, prog = run_local(S, KW, STEPS, batch_fn)
    shards, workers, per_step = simulate(S, STEPS, KW, batch_fn)
    for step in range(STEPS):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"S={S} step {step} worker {r}")
    keys = all_keys(S, STEPS, batch_fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        assert (own == s).sum() > 10
        check_shard(engines[s], shards[s], keys[own == s], f"S={S} shard {s}")
        # nothing leaked to the wrong shard
        if S > 1:
            _, hasv, _, _ = engines[s].read_entries(keys[own != s][:64])
            assert np.all(hasv == -1)
    for E in engines:
        E.close()


def test_fused_shard_equals_single_engine_raw_step():
    """S = 1 through the shard path == the fused single-GPU raw step, same inputs"""
    engines, prog = run_local(1, KW, STEPS, batch_fn)
    E2 = capi.Engine(device=0, table_capacity=1 << 14, **KW)
    for step in range(STEPS):
        off, idx, val, lab = batch_fn(0, step)
        pr2 = E2.train_step_raw(off, idx, val, lab, push_cnt=step < 2, is_train=True)
        assert abs(prog[0][step].loss - pr2.loss) <= 1e-5 * abs(pr2.loss) + 1e-5
        assert abs(prog[0][step].penalty - pr2.penalty) <= 1e-5 * abs(pr2.penalty) + 1e-6
    keys = all_keys(1, STEPS, batch_fn)
    for a, b in zip(engines[0].read_entries(keys), E2.read_entries(keys)):
        assert_close(a, b, what="shard(S=1) vs fused raw step", rtol=1e-5, atol=1e-6)
    assert engines[0].rng_state() == E2.rng_state()


def test_fused_shard_validation_steps_do_not_touch_the_model():
    S = 2
    train_fn = lambda step: step % 3 != 2      # noqa: E731  every third batch is a validation batch
    engines, prog = run_local(S, KW, STEPS, batch_fn, train_fn=train_fn)
    shards, workers, per_step = simulate(S, STEPS, KW, batch_fn, train_fn=train_fn)
    for step in range(STEPS):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"step {step} worker {r}")
    keys = all_keys(S, STEPS, batch_fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        # a validation batch must not insert its unseen keys (the oracle's Get() default-constructs them: compare values)
        scal, hasv, V, cg = engines[s].read_entries(keys[own == s])
        oscal, ohasv, oV, ocg = oracle_state(shards[s].M, keys[own == s])
        seen = hasv >= 0
        assert np.array_equal(hasv[seen], ohasv[seen])
        assert_close(scal[seen][:, 1:], oscal[seen][:, 1:], what="w/sqrt_g/z", **STATE_TOL)
        assert_close(V[seen], oV[seen], what="V", **STATE_TOL)
        assert np.all(oscal[~seen] == 0)


def test_fused_shard_hot_shared_keys_and_v64():
    """few distinct ids: every key is held by every worker in every step (the pull-time V of a key another
    worker's push already updated must be used), V_dim = 64, long column lists"""
    kw = dict(KW, V_dim=64, V_threshold=0)
    fn = lambda rank, step: raw_batch(rank, step, valued=(step % 2 == 1), B=128, ids=40, max_nnz=30)   # noqa: E731
    S, steps = 3, 5
    engines, prog = run_local(S, kw, steps, fn)
    shards, workers, per_step = simulate(S, steps, kw, fn)
    for step in range(steps):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"step {step} worker {r}")
    keys = all_keys(S, steps, fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        check_shard(engines[s], shards[s], keys[own == s], f"shard {s}")


def test_fused_shard_mixed_binary_valued_and_empty_batches():
    """the workers of one step hold a binary batch, a valued one and none at all (the last round of an epoch whose
    file parts have unequal lengths): on the wire every batch is valued, so an owner never has to know"""
    def fn(rank, step):
        if rank == 1 and step in (2, 5):
            return raw_batch(rank, step, valued=False, B=0)
        if rank == 2 and step == 5:
            return raw_batch(rank, step, valued=True, B=0)
        return raw_batch(rank, step, valued=(rank + step) % 2 == 0)
    S = 3
    engines, prog = run_local(S, KW, STEPS, fn)
    shards, workers, per_step = simulate(S, STEPS, KW, fn)
    for step in range(STEPS):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"step {step} worker {r}")
    keys = all_keys(S, STEPS, fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        check_shard(engines[s], shards[s], keys[own == s], f"shard {s}")
    for E in engines:
        E.close()


# ---------------------------------------------------------------------------------------------------------
# dropped worker batches: nothing changes on any owner, nothing is added to that rank's Progress, and the error is
# reported once, by that rank's read of its own step.  The other ranks step as if the worker held an empty batch.
# (new_keys / new_vrows of a rank count its inserts as an OWNER, for every worker's keys: not the dropped batch's.)
# ---------------------------------------------------------------------------------------------------------
PROGRESS = ("loss", "penalty", "auc", "nrows", "new_keys", "new_vrows")
WORKER = ("loss", "penalty", "auc", "nrows")
ZERO = (0.0,) * 4 + (0, 0)


def run_pipelined(engines, fn, steps):
    """step t + 1 is enqueued before step t is read.  Returns per rank and step (rc, Progress, error message)"""
    out = [[] for _ in engines]

    def read(t):
        for r, E in enumerate(engines):
            pr = capi.Progress()
            rc = E.L.dfb_wait_step(E.h, C.byref(pr))
            out[r].append((rc, pr, E.L.dfb_last_error(E.h).decode() if rc else ""))
    for t in range(steps):
        enqueue_local(engines, [fn(r, t) for r in range(len(engines))], t < 2, True)
        if t:
            read(t - 1)
    read(steps - 1)
    for E in engines:
        E.sync()
        assert tuple(getattr(E.read_progress(), f) for f in PROGRESS) == ZERO       # nothing left behind
    return out


def check_dropped(engines, out, kw, steps, fn, fn_sim, bad, code, what):
    """out of run_pipelined; bad = (rank, step) of the dropped batch, code its error.  Returns the error message"""
    S = len(engines)
    prog = [[pr for _, pr, _ in o] for o in out]
    msg = None
    for r in range(S):
        for t in range(steps):
            rc, pr, m = out[r][t]
            if (r, t) == bad:
                assert rc == code, f"{what}: rank {r} step {t}: rc {rc} ({m})"
                assert tuple(getattr(pr, f) for f in WORKER) == ZERO[:4], f"{what}: Progress of the dropped batch"
                msg = m
            else:
                assert rc == 0, f"{what}: rank {r} step {t}: rc {rc} ({m})"
    check_vs_simulation(engines, prog, kw, steps, fn_sim, what)
    own_keys = all_keys(S, steps, fn_sim)
    dropped_only = np.setdiff1d(O.localize(*fn(*bad)[:2])[1], own_keys)
    assert len(dropped_only)
    for E in engines:
        assert np.all(E.read_entries(dropped_only)[1] == -1), f"{what}: a key of the dropped batch was inserted"
    return msg


def rand_ids(rng, n, bits):
    x = (rng.integers(0, 1 << 32, n, dtype=np.uint64) << np.uint64(32)) | rng.integers(0, 1 << 32, n, dtype=np.uint64)
    return x & np.uint64((1 << bits) - 1)


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("id_bits", [16, 30, 36, None])
def test_fused_shard_batch_outside_id_range_is_dropped(id_bits, S):
    """id_bits 16 / 30 (32-bit sort keys), 36 (64-bit), None (the range learned from the first batch: ids below 2^12).
    Rank 1's batch of step 2 carries one id above the range (id_bits: 2^nibble_top, the smallest id outside it;
    learned: ids of 40 bits)"""
    bits = id_bits or 12
    top = 4 * ((bits + 3) // 4)
    pool = np.unique(rand_ids(np.random.default_rng(bits), 3000, bits))
    steps, bad = 5, (1, 2)

    def legal(rank, step):
        rng = np.random.default_rng(10 * rank + step + 100 * bits)
        lens = rng.integers(0, 30, 120)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        idx = pool[rng.integers(0, len(pool), int(off[-1]))]
        val = rng.random(len(idx)).astype(np.float32) if (rank + step) % 2 else None
        lab = np.where(rng.random(120) < 0.4, 1.0, -1.0).astype(np.float32)
        return off, idx, val, lab

    def fn(rank, step):
        off, idx, val, lab = legal(rank, step)
        if (rank, step) != bad:
            return off, idx, val, lab
        idx = idx.copy()
        if id_bits:
            idx[-1] = np.uint64(1 << top)
        else:
            idx[::3] = rand_ids(np.random.default_rng(7), len(idx[::3]), 40) | np.uint64(1 << 39)
        return off, idx, val, lab

    def fn_sim(rank, step):
        return raw_batch(rank, step, valued=False, B=0) if (rank, step) == bad else fn(rank, step)
    kw = dict(KW, V_dim=32)
    engines = make_local(S, kw, engine_kw=dict(id_bits=id_bits) if id_bits else None, max_nnz=8192)
    out = run_pipelined(engines, fn, steps)
    msg = check_dropped(engines, out, kw, steps, fn, fn_sim, bad, capi.DFB_ERR_INVALID, f"id_bits={id_bits} S={S}")
    assert "id_bits = %d" % (id_bits or 0) in msg, msg
    if id_bits:
        assert "2^%d" % top in msg, msg


def test_fused_shard_segment_capacity_is_reported():
    """a key segment larger than seg_keys on rank 1 in step 2 of 4 drops that batch alone, reported with its step"""
    steps, bad = 4, (1, 2)

    def fn(rank, step):     # 60 ids: at most 60 keys per owner segment; the bad batch has ~500 over 2 owners
        return raw_batch(rank, step, valued=step % 2 == 0, ids=500 if (rank, step) == bad else 60)

    def fn_sim(rank, step):
        return raw_batch(rank, step, valued=False, B=0) if (rank, step) == bad else fn(rank, step)
    engines = make_local(2, KW, max_rows=128, max_nnz=4096, seg_keys=64, seg_nnz=2048)
    out = run_pipelined(engines, fn, steps)
    check_dropped(engines, out, KW, steps, fn, fn_sim, bad, capi.DFB_ERR_CAPACITY, "segment capacity")


def test_fused_shard_rows_without_nonzeros_count():
    """a worker batch with rows but no nonzeros is not dropped: its rows count, with prediction 0"""
    def fn(rank, step):
        if rank == 1 and step in (1, 2):
            off, idx, val, lab = raw_batch(rank, step, valued=step == 2, B=40)
            return np.zeros_like(off), idx[:0], None if val is None else val[:0], lab
        return batch_fn(rank, step)
    engines, prog = run_local(2, KW, 4, fn)
    check_vs_simulation(engines, prog, KW, 4, fn, "rows without nonzeros")
    assert prog[1][1].nrows == 40 and prog[1][2].nrows == 40


def test_fused_shard_begin_restages_a_prefetch_with_another_label():
    """a batch prefetched with label array A and begun with the same ids but label array B trains on B: a prefetch is
    reused only for the same pointers, label included.  Compared with a twin store stepped on B without a prefetch"""
    (E,), (T,) = make_local(1, KW), make_local(1, KW)
    off, ids, val, lab = batch_fn(0, 0)
    flipped = -lab
    for X in (E, T):          # a trained model, so that the two labelings give different losses and updates
        enqueue_local([X], [(off, ids, val, lab)], True, True)
        X.wait_step()
    E.prefetch_raw(len(lab), off, ids, val, lab)
    E.shard_begin_async(len(lab), off, ids, val, flipped)
    for phase in range(5):
        E.shard_phase(phase)
    enqueue_local([T], [(off, ids, val, flipped)], False, True)
    pe, pt = E.wait_step(), T.wait_step()
    assert abs(pe.loss - pt.loss) <= 1e-5 * abs(pt.loss) + 1e-5, (pe.loss, pt.loss)
    keys = np.unique(ids)
    for a, b in zip(E.read_entries(keys), T.read_entries(keys)):
        assert_close(a, b, what="prefetch with label A, step on label B", rtol=1e-5, atol=1e-6)
    E.close()
    T.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (gpurun --gpus 2)")
@pytest.mark.parametrize("big", [False, True])
def test_fused_shard_two_gpus_one_process_vs_oracle_simulation(big):
    """two engines on two devices inside ONE process, driven by ONE host thread (peer access instead of CUDA IPC; the
    C++ CLI's num_gpus mode).  The enqueue phases are interleaved over the ranks as on one device: a monolithic
    dfb_shard_step_async per rank would leave rank 0's pollers waiting for work the host has not enqueued yet, and any
    blocking driver call in between (a lazily loaded kernel, for one) then never returns.  big = the CLI's capacities"""
    S = 2
    shard_kw = dict(max_rows=65536, max_nnz=65536 * 64) if big else {}
    engines, prog = run_local(S, KW, STEPS, batch_fn, devices=[0, 1], **shard_kw)
    shards, workers, per_step = simulate(S, STEPS, KW, batch_fn)
    for step in range(STEPS):
        for r in range(S):
            check_progress(prog[r][step], per_step[step][r], f"step {step} worker {r}")
    keys = all_keys(S, STEPS, batch_fn)
    own = key_owner_np(keys, S)
    for s in range(S):
        check_shard(engines[s], shards[s], keys[own == s], f"shard {s}")
    for E in engines:
        E.close()


# ---------------------------------------------------------------------------------------------------------
# one process per GPU, mailboxes shared through CUDA IPC
# ---------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from difacto_b200 import capi as C2
    from difacto_b200.sharded import FusedShardedStore
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    E = C2.Engine(device=rank, table_capacity=1 << 14, **KW)
    store = FusedShardedStore(E, max_rows=128, max_nnz=4096)
    prog = []
    for step in range(STEPS):
        off, idx, val, lab = batch_fn(rank, step)
        store.step_host(len(lab), off, idx, val, lab, is_train=True, push_cnt=step < 2)
        pr = E.wait_step()
        prog.append([pr.loss, pr.penalty, pr.auc, 0.0, pr.nrows])
    keys = all_keys(world, STEPS, batch_fn)
    mine = keys[key_owner_np(keys, world) == rank]
    scal, hasv, V, cg = E.read_entries(mine)
    np.savez(out.format(rank=rank), scal=scal, hasv=hasv, V=V, cg=cg, prog=np.array(prog), nkeys=E.table_stats()["n_keys"])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs (gpurun --gpus 2)")
def test_fused_shard_two_gpus_ipc_vs_oracle_simulation(tmp_path):
    import torch.multiprocessing as mp
    world = 2
    out = str(tmp_path / "shard{rank}.npz")
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    shards, workers, per_step = simulate(world, STEPS, KW, batch_fn)
    keys = all_keys(world, STEPS, batch_fn)
    own = key_owner_np(keys, world)
    for s in range(world):
        got = np.load(out.format(rank=s))
        oscal, ohasv, oV, ocg = oracle_state(shards[s].M, keys[own == s])
        assert np.array_equal(got["hasv"], ohasv)
        assert np.array_equal(got["scal"][:, 0], oscal[:, 0])
        assert_close(got["scal"][:, 1:], oscal[:, 1:], what=f"shard {s} w/sqrt_g/z", **STATE_TOL)
        assert_close(got["V"], oV, what=f"shard {s} V", **STATE_TOL)
        assert_close(got["cg"], ocg, what=f"shard {s} cg", **STATE_TOL)
        assert got["nkeys"] == shards[s].M.size()
        for step in range(STEPS):
            ref = per_step[step][s]
            assert abs(got["prog"][step][0] - ref[0]) <= 1e-4 * abs(ref[0]) + 1e-4
            assert abs(got["prog"][step][1] - ref[1]) <= 1e-4 * abs(ref[1]) + 1e-5
