"""The raw training step without a key lookup: a sorted training step on raw ids without a feature-count push, whose
pulled view would not fit in L2 (V_dim > 0, l2_hints on), probes the table with each nonzero's id in the forward and
finds or inserts every key in the update.  Smaller batches still run the lookup, and their update takes its slots.
Sequences of raw steps (dfb_train_step_raw_dev) must leave exactly what a twin engine leaves that is fed the same
batches through the host-localized dfb_train_step, which looks every key up first: the same table entries, V rows,
AdaGrad state, table counts and rand_r state, and the same Progress of every step.

Covered: V_dim 0 ... 128 (padded and exact lane widths), binary and valued batches, rows at and above long_row_nnz,
keys over hot_split, a cold first step (every key inserted by the update), push_cnt, validation and predict steps
between training steps, a table just large enough for the keys (long probe chains), a table too small for a batch
(DFB_ERR_CAPACITY from the same step on both engines) and a batch dropped for its id range -- on batches small enough
to keep the lookup, and on batches above the L2 bound, which run without it (checked from the profiled lookup stage)."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_id_range as idr
from util import localized

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=2, V_l2=0.02, V_init_scale=0.2, seed=11)
ENGINE = dict(long_row_nnz=200, hot_split=64)


def batch(rng, pool, B=500, valued=False, hot=None):
    """rows of 0..40 ids from pool, three rows of 200..300 ids (k_fm_long's), and optionally id `hot` in 300 rows
    (an occurrence list above hot_split: pre-reduced in chunks)"""
    lens = rng.integers(0, 41, B)
    lens[rng.choice(B, 3, replace=False)] = rng.integers(200, 301, 3)
    rows = [pool[rng.integers(0, len(pool), n)] for n in lens]
    if hot is not None:
        for r in rng.choice(B, 300, replace=False):
            rows[r] = np.concatenate([rows[r], np.array([hot], U64)])
    ids = np.concatenate(rows).astype(U64)
    return idr.csr(rng, np.array([len(r) for r in rows]), ids, valued)


def train_pair(E, T, b, push, dev):
    """one training step on both engines: (rc, Progress) of each"""
    o, l, i, v = b
    do, dl, di, dv = dev
    E.train_step_raw_dev(len(l), len(i), do, di, dv, dl, push, True)
    re, pe = idr.progress_rc(E, "dfb_read_progress")
    loc = localized(b)
    pt = capi.Progress()
    rt = T.L.dfb_train_step(T.h, len(l), capi._p(o), capi._p(loc["lidx"]), capi._p(v), capi._p(l),
                            capi._p(loc["keys"]), len(loc["keys"]), capi._p(loc["cnt"] if push else None), 1,
                            C.byref(pt), None)
    return (re, pe), (rt, pt)


def run_sequence(E, T, batches, plan, model_every_step=True):
    """plan: (kind, batch index, push_cnt) with kind train / val / predict; every step is compared on both engines"""
    dev = [idr.on_device(b) for b in batches]
    seen = []
    for t, (kind, j, push) in enumerate(plan):
        b = batches[j]
        o, l, i, v = b
        if kind == "train":
            (re, pe), (rt, pt) = train_pair(E, T, b, push, dev[j])
            assert re == 0 and rt == 0, (t, E.L.dfb_last_error(E.h).decode())
            assert idr.as_tuple(pe) == idr.as_tuple(pt), (t, kind, idr.as_tuple(pe), idr.as_tuple(pt))
            seen.append(b)
        elif kind == "val":
            do, dl, di, dv = dev[j]
            E.train_step_raw_dev(len(l), len(i), do, di, dv, dl, False, False)
            pe = E.read_progress()
            loc = localized(b)
            pt = T.train_step(o, loc["lidx"], v, l, loc["keys"], None, False)
            assert idr.as_tuple(pe) == idr.as_tuple(pt), (t, kind)
        else:
            pe, qe = E.predict_raw(o, i, v, l)
            pt, qt = T.predict_raw(o, i, v, l)
            assert np.array_equal(qe, qt) and idr.as_tuple(pe) == idr.as_tuple(pt), (t, kind)
        if seen and (model_every_step or t == len(plan) - 1):
            idr.assert_same_model(E, T, idr.seen_keys(seen + [b]))
    return seen


@pytest.mark.parametrize("V_dim", [0, 1, 10, 16, 40, 64, 100, 128])
@pytest.mark.parametrize("valued", [False, True])
def test_raw_steps_equal_host_localized_steps(V_dim, valued):
    rng = np.random.default_rng(31 * V_dim + valued)
    pool = np.unique(rng.integers(0, 1 << 40, 4000).astype(U64) * GOLDEN)
    batches = [batch(rng, pool[:1500], valued=valued, hot=pool[7]),        # cold: every key is new
               batch(rng, pool[1000:3000], valued=valued, hot=pool[7]),    # half of the keys new
               batch(rng, pool, valued=valued),
               batch(rng, pool[3000:], valued=valued, hot=pool[3100]),
               batch(rng, np.concatenate([pool, pool[:500] + U64(1)]), valued=valued)]   # ids the table never saw
    kw = dict(V_dim=V_dim, table_capacity=1 << 14, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    plan = [("train", 0, False), ("train", 1, False), ("val", 2, False), ("train", 2, True), ("predict", 4, False),
            ("train", 3, False), ("train", 0, False), ("val", 4, False), ("train", 4, False), ("train", 1, True),
            ("predict", 3, False), ("train", 2, False)]
    run_sequence(E, T, batches, plan)
    st = E.table_stats()
    assert V_dim == 0 or 0 < st["n_vrows"] < st["n_keys"]          # keys with and without V rows


@pytest.mark.parametrize("valued", [False, True])
def test_full_table_long_probe_chains(valued):
    """a table sized just above the keys it will hold: half of its slots taken, the insert / find chains long"""
    rng = np.random.default_rng(5 + valued)
    pool = np.unique(rng.integers(0, 1 << 40, 4096).astype(U64) * GOLDEN)
    batches = [batch(rng, pool[:2000], B=900, valued=valued), batch(rng, pool[1500:], B=900, valued=valued),
               batch(rng, pool, B=900, valued=valued)]
    n = len(idr.seen_keys(batches))
    kw = dict(V_dim=16, table_capacity=n + 8, V_capacity=n + 8, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    run_sequence(E, T, batches, [("train", 0, False), ("train", 1, False), ("train", 2, False), ("train", 0, True),
                                 ("train", 2, False)])
    assert E.table_stats()["n_keys"] == n


def test_table_too_small_reports_capacity_in_the_same_step():
    rng = np.random.default_rng(9)
    pool = np.unique(rng.integers(0, 1 << 40, 3000).astype(U64) * GOLDEN)
    small, large = batch(rng, pool[:300], B=200), batch(rng, pool[:1500], B=800)
    # more keys than table_capacity, but fewer than the 2048 slots of the table: every key is inserted on both engines
    assert len(idr.seen_keys([small])) < 1000 < len(idr.seen_keys([large])) < 2000
    kw = dict(V_dim=16, table_capacity=1000, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    for t, (b, want) in enumerate([(small, 0), (large, capi.DFB_ERR_CAPACITY), (small, 0)]):
        (re, pe), (rt, pt) = train_pair(E, T, b, False, idr.on_device(b))
        assert re == want and rt == want, (t, re, rt)
        if want == 0:
            assert idr.as_tuple(pe) == idr.as_tuple(pt), t
    idr.assert_same_model(E, T, idr.seen_keys([small, large]))


def test_dropped_batch_changes_nothing_and_is_reported_once():
    rng = np.random.default_rng(13)
    pool = np.unique(idr.rand_u64(rng, 3000, 30))
    good = [batch(rng, pool, B=300, valued=j == 1) for j in range(3)]
    o, l, i, v = batch(rng, pool, B=300)
    bad = idr.csr(rng, np.diff(o.astype(np.int64)) + np.eye(len(l), dtype=np.int64)[-1],
                  np.concatenate([i, np.array([1 << 32], U64)]), False)      # one id above the sorted range
    kw = dict(V_dim=64, id_bits=30, table_capacity=1 << 14, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    run_sequence(E, T, good, [("train", 0, False), ("train", 1, False)])
    do, dl, di, dv = idr.on_device(bad)
    E.train_step_raw_dev(len(bad[1]), len(bad[2]), do, di, dv, dl, False, True)
    rc, pr = idr.progress_rc(E, "dfb_read_progress")
    assert rc == capi.DFB_ERR_INVALID and "id_bits = 30" in E.L.dfb_last_error(E.h).decode()
    assert idr.as_tuple(pr) == (0.0,) * 4 + (0, 0)
    assert idr.as_tuple(E.read_progress()) == (0.0,) * 4 + (0, 0)
    idr.assert_same_model(E, T, idr.seen_keys(good + [bad]))
    run_sequence(E, T, good, [("train", 2, False), ("train", 0, False)])


def big_batch(rng, pool, rows, valued, hot=None):
    """rows of 30..70 ids from pool (over 3.3 M nonzeros: a pulled view of that bound does not fit in half an H100's L2),
    three rows of 200..300 ids, `hot` as the first id of 400 rows"""
    lens = rng.integers(30, 71, rows)
    lens[rng.choice(rows, 3, replace=False)] = rng.integers(200, 301, 3)
    ids = pool[rng.integers(0, len(pool), int(lens.sum()))]
    if hot is not None:
        starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
        ids[starts[rng.choice(rows, 400, replace=False)]] = hot
    return idr.csr(rng, lens, ids, valued)


def above_l2_bound(batches):
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    return all(len(b[2]) * 8 > l2 // 2 for b in batches)


def lookup_stage_ms(E, b, is_train):
    """the profiled lookup stage (stage 0) of one raw step of E on batch b, in ms (a training step changes E)"""
    do, dl, di, dv = idr.on_device(b)
    E.sync()
    E.profile(True)
    E.train_step_raw_dev(len(b[1]), len(b[2]), do, di, dv, dl, False, is_train)
    E.sync()
    st = E.profile_read()["lookup"]
    E.profile(False)
    E.read_progress()
    assert st["count"] == 1
    return st["ms"]


def assert_ran_without_lookup(E, b):
    """a training step on b has an empty lookup stage, where the validation step on b runs k_lookup over its keys"""
    val = lookup_stage_ms(E, b, False)
    train = lookup_stage_ms(E, b, True)
    assert train < 0.2 * val, (train, val)


@pytest.mark.parametrize("V_dim,valued", [(1, False), (10, True), (16, False), (64, False), (64, True), (128, False)])
def test_large_batches_run_without_lookup_and_equal_host_localized_steps(V_dim, valued):
    rng = np.random.default_rng(77 + V_dim + valued)
    pool = np.unique(rng.integers(0, 1 << 40, 700000).astype(U64) * GOLDEN)
    batches = [big_batch(rng, pool[:400000], 70000, valued, pool[3]),            # cold: every key is new
               big_batch(rng, pool[200000:], 70000, valued, pool[3]),
               big_batch(rng, np.concatenate([pool, pool[:100000] + U64(1)]), 70000, valued, pool[5])]
    assert above_l2_bound(batches)
    kw = dict(V_dim=V_dim, table_capacity=1 << 20, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    plan = [("train", 0, False), ("train", 1, False), ("val", 2, False), ("train", 1, True), ("predict", 2, False),
            ("train", 2, False), ("train", 0, False)]
    run_sequence(E, T, batches, plan, model_every_step=False)
    assert_ran_without_lookup(E, batches[1])


def test_large_batches_full_table_long_probe_chains():
    """a table whose slots the keys fill to just under one half: long insert / find chains on the lookup-free path"""
    rng = np.random.default_rng(21)
    pool = np.unique(rng.integers(0, 1 << 40, 524100).astype(U64) * GOLDEN)[:524000]
    batches = [big_batch(rng, pool, 70000, False), big_batch(rng, pool, 70000, True)]
    assert above_l2_bound(batches)
    n = len(idr.seen_keys(batches))
    assert 2 * n + 16 <= 1 << 20 < 4 * n                 # 2^20 slots, more than 49 % of them taken
    kw = dict(V_dim=16, table_capacity=n + 8, V_capacity=n + 8, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    run_sequence(E, T, batches, [("train", 0, False), ("train", 1, False), ("train", 0, True), ("train", 1, False)],
                 model_every_step=False)
    assert E.table_stats()["n_keys"] == n
    assert_ran_without_lookup(E, batches[0])


def test_large_batch_over_table_capacity_reports_it_in_the_same_step():
    rng = np.random.default_rng(23)
    pool = np.unique(rng.integers(0, 1 << 40, 400000).astype(U64) * GOLDEN)
    small, large = big_batch(rng, pool[:200000], 70000, False), big_batch(rng, pool, 70000, False)
    assert above_l2_bound([small, large])
    # more keys than table_capacity, fewer than the table's 2^20 slots: every key is inserted on both engines
    assert len(idr.seen_keys([small])) < 300000 < len(idr.seen_keys([large])) < 500000
    kw = dict(V_dim=16, table_capacity=300000, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    for t, (b, want) in enumerate([(small, 0), (large, capi.DFB_ERR_CAPACITY), (small, 0)]):
        (re, pe), (rt, pt) = train_pair(E, T, b, False, idr.on_device(b))
        assert re == want and rt == want, (t, re, rt)
        if want == 0:
            assert idr.as_tuple(pe) == idr.as_tuple(pt), t
    idr.assert_same_model(E, T, idr.seen_keys([small, large]))
    assert_ran_without_lookup(E, small)


def test_large_batch_outside_id_bits_is_dropped_without_lookup():
    rng = np.random.default_rng(25)
    pool = np.unique(idr.rand_u64(rng, 400000, 24))
    good = [big_batch(rng, pool, 70000, j == 1) for j in range(3)]
    o, l, i, v = big_batch(rng, pool, 70000, False)
    bad = idr.csr(rng, np.diff(o.astype(np.int64)) + np.eye(len(l), dtype=np.int64)[-1],
                  np.concatenate([i, np.array([1 << 24], U64)]), False)      # one id above the sorted range
    assert above_l2_bound(good + [bad])
    kw = dict(V_dim=64, id_bits=24, table_capacity=1 << 20, **ENGINE, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    run_sequence(E, T, good, [("train", 0, False), ("train", 1, False)], model_every_step=False)
    do, dl, di, dv = idr.on_device(bad)
    E.train_step_raw_dev(len(bad[1]), len(bad[2]), do, di, dv, dl, False, True)
    rc, pr = idr.progress_rc(E, "dfb_read_progress")
    assert rc == capi.DFB_ERR_INVALID and "id_bits = 24" in E.L.dfb_last_error(E.h).decode()
    assert idr.as_tuple(pr) == (0.0,) * 4 + (0, 0)
    assert idr.as_tuple(E.read_progress()) == (0.0,) * 4 + (0, 0)
    idr.assert_same_model(E, T, idr.seen_keys(good + [bad]))
    run_sequence(E, T, good, [("train", 2, False), ("train", 0, False)], model_every_step=False)
    assert_ran_without_lookup(E, good[2])
