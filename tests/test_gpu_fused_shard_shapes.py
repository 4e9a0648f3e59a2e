"""The NVLink-sharded store (dfb_shard_*) at the shapes the benchmark runs it, against tests/shard_sim.simulate.

All ranks share one GPU (engines of one process, phases interleaved as in shard_sim.run_local).  Cases:
  * every V_dim (8..128), binary and valued, S = 2 and 3: every K instantiation of k_fm_fast<K,3>, k_shard_reduce<K>,
    k_shard_pull and k_bwd_update<K,.,.,SRC=2>.  Rows are empty, one 32-nonzero chunk, several, or 1024..1500 long;
    one id sits in every other row of a worker's batch and one in every third row of every worker's batch, so the
    owner pre-reduces their column lists in chunks (hot_split) and the shared one also carries a pull-time V row;
  * a worker batch of 2 x 8192 + 13 rows: k_shard_rowscan carries its prefix over 1024 x 8-row blocks;
  * hot_split 16 and the default 256 on the owner;
  * the benchmark's own batches (bench.gen_raw_batch) and hyper-parameters (bench.hyper): criteo39 with full-size
    segments (criteo_conf, allV, ftrl_l1) and the synthetic workload with id_bits = 30;
  * reversed keys at the ownership boundaries w*s - 1, w*s, w*s + 1 (w = ~0 / S) and the largest key, S = 2, 3, 4;
  * bit-for-bit invariance: a second run, l2_hints 0 / 1;
  * S = 1 against the single-GPU raw step at every V_dim.
Tolerances as in test_gpu_fused_shard.py (shard_sim.STATE_TOL, check_progress: loss 1e-4 relative), with two
exceptions (LOOSE) that come from column lists hundreds of rows long: the simulation adds their gradients up in
float32, in row order, while the owner adds them in chunks.  The penalty of the steps after the first, a sum over
thousands of keys of l1 |w| + l2 w^2 + V_l2 |V|^2, moved by up to 4.4e-4 relative on an H100 (V_dim 128); and V
entries near zero by up to 1.6e-5 absolute (1 entry in ~10^5).  At most 4 ranks share the GPU:
each engine uses 7 streams, and CUDA_DEVICE_MAX_CONNECTIONS=32 gives 4 ranks a hardware queue per stream."""
import argparse
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from oracle import oracle as O  # noqa: E402
from shard_sim import (HOT_SHARED, all_keys, check_vs_simulation, hot_own, key_owner_np, raw_batch,  # noqa: E402
                       run_local)
from util import assert_close  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)
U64 = np.uint64
# mixed / hot batches: ~47k nonzeros, ~900 rows, both hot ids well over 256 occurrences per worker batch
MIXED = dict(B=900, ids=3000, mixed=True, hot=True)
MIXED_CAP = dict(max_rows=1024, max_nnz=1 << 16)
LOOSE = dict(pen_rtol=2e-3, state_tol=dict(rtol=1e-3, atol=5e-5))


def mixed_fn(valued=None):
    """valued None: binary and valued batches alternate over ranks and steps"""
    def fn(rank, step):
        v = (rank + step) % 2 == 0 if valued is None else valued
        return raw_batch(rank, step, valued=v, **MIXED)
    return fn


def test_mixed_batches_reach_every_loop():
    off, idx, _, _ = raw_batch(0, 0, valued=False, **MIXED)
    lens = np.diff(off.astype(np.int64))
    assert (lens == 0).any() and ((lens > 0) & (lens < 32)).any() and ((lens > 32) & (lens <= 200)).any()
    assert (lens >= 1024).sum() == 3
    assert (idx == hot_own(0)).sum() > 256 and (idx == HOT_SHARED).sum() > 256


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("valued", [False, True])
@pytest.mark.parametrize("K", [8, 16, 32, 64, 128])
def test_every_vdim_long_rows_hot_keys_vs_simulation(K, valued, S):
    kw = dict(KW, V_dim=K)
    fn = mixed_fn(valued)
    engines, prog = run_local(S, kw, 3, fn, **MIXED_CAP)
    check_vs_simulation(engines, prog, kw, 3, fn, f"K={K} valued={valued} S={S}", **LOOSE)


@pytest.mark.parametrize("S", [2, 3])
def test_worker_batch_past_one_rowscan_block(S):
    """worker 0 holds 2 x 8192 + 13 rows (= max_rows, not a multiple of 8), the others fewer"""
    B0 = 2 * 8192 + 13
    kw = dict(KW, V_dim=32)

    def fn(rank, step):
        return raw_batch(rank, step, valued=step % 2 == 1, B=B0 if rank == 0 else 5000 + 777 * rank, ids=4000,
                         max_nnz=7)
    engines, prog = run_local(S, kw, 3, fn, engine_kw=dict(table_capacity=1 << 15), max_rows=B0, max_nnz=8 * B0)
    check_vs_simulation(engines, prog, kw, 3, fn, f"S={S}", **LOOSE)
    assert prog[0][0].nrows == B0


@pytest.mark.parametrize("hot_split", [16, 256])
def test_owner_hot_split_vs_simulation(hot_split):
    kw = dict(KW, V_dim=64)
    fn = mixed_fn()
    assert max((fn(r, 0)[1] == HOT_SHARED).sum() for r in range(3)) > 256
    engines, prog = run_local(3, kw, 3, fn, engine_kw=dict(hot_split=hot_split), **MIXED_CAP)
    check_vs_simulation(engines, prog, kw, 3, fn, f"hot_split={hot_split}", **LOOSE)


# ---------------------------------------------------------------------------------------------------------------------
# the benchmark's batches and hyper-parameters
# ---------------------------------------------------------------------------------------------------------------------
def bench_args(workload, hyper, vdim, rows):
    return argparse.Namespace(workload=workload, hyper=hyper, vdim=vdim, batch=rows, nnz=100, id_space=10 ** 9)


def bench_fn(args):
    cache = {}

    def fn(rank, step):
        if (rank, step) not in cache:
            off, lab, ids, val = bench.gen_raw_batch(args, 1 + 1000 * rank + step)
            cache[(rank, step)] = (off, ids, val, lab)
        return cache[(rank, step)]
    return fn


@pytest.mark.parametrize("hyper,vdim", [("criteo_conf", 64), ("allV", 64), ("ftrl_l1", 32)])
def test_bench_criteo39_vs_simulation(hyper, vdim):
    """criteo39 rows (the group in the ids' low 12 bits: the reversed keys cluster by owner), full-size segments as
    the benchmark passes them; 8192 rows put the z = 1 id of every group over the owner's hot_split"""
    args = bench_args("criteo39", hyper, vdim, 8192)
    kw = bench.hyper(args)
    fn = bench_fn(args)
    N = 8192 * bench.nnz_of(args)
    for r in range(2):
        _, cnt = np.unique(fn(r, 0)[1], return_counts=True)
        assert cnt.max() > 256
    engines, prog = run_local(2, kw, 2, fn, cnt_steps=1, engine_kw=dict(table_capacity=1 << 20, V_capacity=1 << 20),
                              max_rows=8192, max_nnz=N, seg_keys=N, seg_nnz=N)
    check_vs_simulation(engines, prog, kw, 2, fn, f"criteo39 {hyper}", cnt_steps=1, **LOOSE)


def test_bench_synthetic_id_bits_30_vs_simulation():
    args = bench_args("synthetic", "allV", 64, 1024)
    kw = bench.hyper(args)
    fn = bench_fn(args)
    N = 1024 * 100
    engines, prog = run_local(2, kw, 2, fn, cnt_steps=1,
                              engine_kw=dict(table_capacity=1 << 19, V_capacity=1 << 19, id_bits=30),
                              max_rows=1024, max_nnz=N)
    check_vs_simulation(engines, prog, kw, 2, fn, "synthetic id_bits=30", cnt_steps=1, **LOOSE)


# ---------------------------------------------------------------------------------------------------------------------
# ownership boundaries
# ---------------------------------------------------------------------------------------------------------------------
def boundary_keys(S):
    w = 0xFFFFFFFFFFFFFFFF // S
    ks = [0, 1, 0xFFFFFFFFFFFFFFFE]          # UINT64_MAX marks an empty slot: 2^64 - 2 is the largest key
    for s in range(1, S):
        ks += [w * s - 1, w * s, w * s + 1]
    return np.array(sorted(set(ks)), U64)


@pytest.mark.parametrize("S", [2, 3, 4])
def test_ownership_boundaries_vs_simulation(S):
    """64-bit sort keys (no id_bits, learned range) with keys on both sides of every owner boundary"""
    kw = dict(KW, V_dim=16)
    bkeys = boundary_keys(S)
    bids = O.reverse_bytes_np(bkeys)         # the nibble reversal is its own inverse

    def fn(rank, step):
        off, idx, val, lab = raw_batch(rank, step, valued=step % 2 == 0, B=128)
        idx = idx.copy()
        at = (np.arange(len(bids)) * 7 + rank) % len(idx)
        idx[at] = np.roll(bids, rank + step)
        return off, idx, val, lab
    engines, prog = run_local(S, kw, 3, fn)
    keys, own, _ = check_vs_simulation(engines, prog, kw, 3, fn, f"S={S}")
    bown = key_owner_np(bkeys, S)
    assert [capi.key_owner(int(k), S) for k in bkeys] == bown.tolist()
    assert sorted(set(bown.tolist())) == list(range(S))
    for s in range(S):
        _, hasv, _, _ = engines[s].read_entries(bkeys)
        assert np.array_equal(hasv != -1, bown == s), f"S={S} shard {s}: {hasv} {bown}"


# ---------------------------------------------------------------------------------------------------------------------
# bit-for-bit invariance
# ---------------------------------------------------------------------------------------------------------------------
PROGRESS = ("loss", "penalty", "auc", "nrows", "new_keys", "new_vrows")


def outcome(engines, prog, keys):
    return ([[tuple(getattr(p, f) for f in PROGRESS) for p in pr] for pr in prog],
            [E.read_entries(keys) for E in engines], [E.rng_state() for E in engines],
            [E.table_stats() for E in engines])


def assert_same(a, b, what):
    assert a[0] == b[0], f"{what}: Progress"
    for ea, eb in zip(a[1], b[1]):
        for x, y in zip(ea, eb):
            assert np.array_equal(x, y), f"{what}: entries"
    assert a[2] == b[2] and a[3] == b[3], f"{what}: rng state / table"


def test_bit_identical_across_runs_and_l2_hints():
    kw = dict(KW, V_dim=64)
    fn = mixed_fn()
    S, steps = 2, 3
    keys = all_keys(S, steps, fn)
    runs = {}
    for name, ekw in (("hints", dict(l2_hints=1)), ("again", dict(l2_hints=1)), ("no hints", dict(l2_hints=0))):
        engines, prog = run_local(S, kw, steps, fn, engine_kw=ekw, **MIXED_CAP)
        runs[name] = outcome(engines, prog, keys)
        if name == "hints":
            check_vs_simulation(engines, prog, kw, steps, fn, name, **LOOSE)
        for E in engines:
            E.close()
    assert_same(runs["hints"], runs["again"], "second run")
    assert_same(runs["hints"], runs["no hints"], "l2_hints=0")


@pytest.mark.parametrize("K", [8, 16, 32, 64, 128])
def test_single_rank_equals_single_engine_raw_step(K):
    """S = 1 through the shard path == the fused single-GPU raw step, same inputs"""
    kw = dict(KW, V_dim=K)

    def fn(rank, step):
        return raw_batch(rank, step, valued=(step % 2 == 0))
    steps = 6
    engines, prog = run_local(1, kw, steps, fn)
    E2 = capi.Engine(device=0, table_capacity=1 << 14, **kw)
    for step in range(steps):
        off, idx, val, lab = fn(0, step)
        pr2 = E2.train_step_raw(off, idx, val, lab, push_cnt=step < 2, is_train=True)
        assert abs(prog[0][step].loss - pr2.loss) <= 1e-5 * abs(pr2.loss) + 1e-5
        assert abs(prog[0][step].penalty - pr2.penalty) <= 1e-5 * abs(pr2.penalty) + 1e-6
        assert prog[0][step].nrows == pr2.nrows
    keys = all_keys(1, steps, fn)
    for a, b in zip(engines[0].read_entries(keys), E2.read_entries(keys)):
        assert_close(a, b, what=f"K={K} shard(S=1) vs fused raw step", rtol=1e-5, atol=1e-6)
    assert engines[0].rng_state() == E2.rng_state()
