"""Capacity growth: an engine created with table_capacity = 1024 and large maxima (table_capacity_max /
V_capacity_max) grows its hash table and V-row pool on demand, and must compute exactly what a pre-sized twin computes:
the same Progress every step, bitwise equal predictions, and at the end the same snapshot bytes and rand_r state.

Covered: raw steps through the synchronous, pipelined (two steps in flight, dfb_prefetch_raw) and device entry
points with push_cnt, validation and predict steps between them, at V_dim 0, 10 and 64, binary and valued; large
batches that take the lookup-free step (the key-finding update on a rehashed table); host-localized dfb_train_step
and the API path; the maxima as hard limits (DFB_ERR_CAPACITY from the same step as a fixed engine of that size);
restore of snapshots larger than the initial capacity, also 2 parts into 3 ranks; that replaced tables are freed;
the parameter checks; the sharded store's refusal; and the CLI."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

import test_gpu_id_range as idr
import test_gpu_lookup_free_step as tlf
from util import localized

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)
# id_bits 64: the ids span all 64 bits, so the pipelined entry points must not learn a narrower range from a first batch
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=2, V_l2=0.02, V_init_scale=0.2, seed=11,
          long_row_nnz=200, hot_split=64, id_bits=64)
GROW = dict(table_capacity=1024, table_capacity_max=1 << 22)
FIXED = dict(table_capacity=1 << 18)


def twins(V_dim, **kw):
    """(growing engine, pre-sized engine) of the same model"""
    return (capi.Engine(V_dim=V_dim, **GROW, **KW, **kw), capi.Engine(V_dim=V_dim, **FIXED, **KW, **kw))


def batches_of(rng, valued, sizes=(200, 400, 800, 1600, 2400)):
    """batches of growing size over a pool of 60000 ids: every step brings new keys"""
    pool = np.unique(rng.integers(0, 1 << 40, 60000).astype(U64) * GOLDEN)
    out = []
    for j, B in enumerate(sizes):
        lo = j * len(pool) // (len(sizes) + 1)
        out.append(tlf.batch(rng, pool[lo:lo + 8 * B + 2000], B=B, valued=valued, hot=pool[lo + 3] if B >= 300 else None))
    return out


def assert_same_end(G, T):
    assert G.snapshot() == T.snapshot()
    assert G.rng_state() == T.rng_state()
    g, t = G.table_stats(), T.table_stats()
    assert (g["n_keys"], g["n_vrows"]) == (t["n_keys"], t["n_vrows"])


PLAN = [("train", 0, True), ("train", 1, False), ("val", 2, False), ("train", 2, False), ("predict", 3, False),
        ("train", 3, True), ("train", 4, False), ("predict", 4, False), ("train", 0, False)]


def run_steps(E, batches, plan, entry, caps=None):
    """the plan on E through one entry point; returns each step's Progress tuple and each predict step's predictions.
    caps (a list) receives the key and V-row capacities after every step."""
    prog, preds, pending = [], [], []
    dev = [idr.on_device(b) for b in batches] if entry == "dev" else None
    keep = []
    for kind, j, push in plan:
        o, l, i, v = batches[j]
        if kind == "predict":
            while pending:
                prog.append(idr.as_tuple(E.wait_step()))
                pending.pop()
            pr, q = E.predict_raw(o, i, v, l)
            prog.append(idr.as_tuple(pr))
            preds.append(q)
        elif entry == "sync":
            prog.append(idr.as_tuple(E.train_step_raw(o, i, v, l, push, kind == "train")))
        elif entry == "dev":
            do, dl, di, dv = dev[j]
            E.train_step_raw_dev(len(l), len(i), do, di, dv, dl, push, kind == "train")
            prog.append(idr.as_tuple(E.read_progress()))
        else:                  # two steps in flight; the next batch is staged before the step is submitted
            keep.append(batches[j])
            E.prefetch_raw(len(l), o, i, v, l)
            E.train_step_raw_async(len(l), o, i, v, l, push, kind == "train")
            pending.append(True)
            if len(pending) == 2:
                prog.append(idr.as_tuple(E.wait_step()))
                pending.pop()
        if caps is not None:   # (waits for the steps in flight, without collecting them)
            st = E.table_stats()
            caps.append((st["capacity"], st["v_capacity"]))
    while pending:
        prog.append(idr.as_tuple(E.wait_step()))
        pending.pop()
    return prog, preds


@pytest.mark.parametrize("entry", ["sync", "async", "dev"])
@pytest.mark.parametrize("V_dim,valued", [(0, False), (10, True), (64, False), (64, True)])
def test_raw_steps_on_a_growing_engine_equal_a_presized_one(entry, V_dim, valued):
    rng = np.random.default_rng(7 * V_dim + valued)
    batches = batches_of(rng, valued)
    G, T = twins(V_dim)
    caps = []
    pg, qg = run_steps(G, batches, PLAN, entry, caps)
    pt, qt = run_steps(T, batches, PLAN, "sync")
    assert pg == pt
    assert all(np.array_equal(a, b) for a, b in zip(qg, qt)) and len(qg) == 2
    assert_same_end(G, T)
    st = G.table_stats()
    assert len(set(c[0] for c in caps)) >= 3, caps           # several table growths ...
    assert st["n_keys"] <= st["capacity"] < T.table_stats()["capacity"]
    if V_dim:
        assert len(set(c[1] for c in caps)) >= 3, caps       # ... and pool growths
        assert 1024 < st["v_capacity"] and st["n_vrows"] <= st["v_capacity"]


def test_lookup_free_steps_on_a_rehashed_table():
    """a small batch first, then 3.5 M-nonzero batches: the table holding the small batch's keys is rehashed before the
    first large step, whose update finds and inserts its keys in the new table"""
    rng = np.random.default_rng(41)
    pool = np.unique(rng.integers(0, 1 << 40, 700000).astype(U64) * GOLDEN)
    batches = [tlf.batch(rng, pool[:3000], B=500),
               tlf.big_batch(rng, pool[:400000], 70000, False, pool[3]),
               tlf.big_batch(rng, pool[200000:], 70000, True, pool[3])]
    assert tlf.above_l2_bound(batches[1:])
    G = capi.Engine(V_dim=16, table_capacity=1024, table_capacity_max=1 << 21, **KW)
    T = capi.Engine(V_dim=16, table_capacity=1 << 21, **KW)
    plan = [("train", 0, False), ("train", 1, False), ("val", 2, False), ("train", 2, False), ("predict", 2, False),
            ("train", 1, False)]
    caps = []
    pg, qg = run_steps(G, batches, plan, "async", caps)
    pt, qt = run_steps(T, batches, plan, "sync")
    assert pg == pt and all(np.array_equal(a, b) for a, b in zip(qg, qt))
    assert caps[0][0] < caps[1][0]                               # grown before the first large step
    assert_same_end(G, T)
    tlf.assert_ran_without_lookup(G, batches[2])


def test_host_localized_steps_and_the_api_path():
    rng = np.random.default_rng(3)
    batches = batches_of(rng, False)
    G, T = twins(10)
    for t, b in enumerate(batches):
        o, l, i, v = b
        loc = localized(b)
        pg = G.train_step(o, loc["lidx"], v, l, loc["keys"], loc["cnt"] if t % 2 == 0 else None, t != 2)
        pt = T.train_step(o, loc["lidx"], v, l, loc["keys"], loc["cnt"] if t % 2 == 0 else None, t != 2)
        assert idr.as_tuple(pg) == idr.as_tuple(pt), t
    # the API path on keys the table has not seen: model_[key] inserts
    keys = np.unique(rng.integers(0, 1 << 40, 30000).astype(U64) * GOLDEN)
    cnt = rng.integers(1, 5, len(keys)).astype(np.float32)
    for E in (G, T):
        E.push_feacnt(keys[:20000], cnt[:20000])
    vg, lg = G.pull(keys)
    vt, lt = T.pull(keys)
    assert np.array_equal(vg, vt) and np.array_equal(lg, lt)
    grads = (rng.random(len(vg)).astype(np.float32) - 0.5)
    for E in (G, T):
        E.push_grad(keys, grads, lg)
    assert np.array_equal(G.pull(keys)[0], T.pull(keys)[0])
    assert_same_end(G, T)
    assert G.table_stats()["capacity"] >= G.table_stats()["n_keys"] > 30000


def raw_rc(E, b):
    """rc and Progress of one synchronous raw training step (the Python wrapper raises on an error)"""
    o, l, i, v = b
    pr = capi.Progress()
    rc = E.L.dfb_train_step_raw(E.h, len(l), capi._p(o), capi._p(i), capi._p(v), capi._p(l), 1, 1, C.byref(pr), None)
    return rc, idr.as_tuple(pr)


@pytest.mark.parametrize("which", ["table", "V"])
def test_the_maxima_are_limits_like_a_fixed_capacity(which):
    rng = np.random.default_rng(17)
    batches = batches_of(rng, False, sizes=(200, 400, 800, 1600, 200))
    kw = dict(KW, V_threshold=0)
    R = capi.Engine(V_dim=10, **FIXED, **kw)       # the counts after each step, without a limit
    counts = []
    for b in batches:
        assert raw_rc(R, b)[0] == 0
        st = R.table_stats()
        counts.append(st["n_keys"] if which == "table" else st["n_vrows"])
    M = (counts[2] + counts[3]) // 2               # the fourth step overflows
    if which == "table":
        G = capi.Engine(V_dim=10, table_capacity=1024, table_capacity_max=M, **kw)
        F = capi.Engine(V_dim=10, table_capacity=M, **kw)
    else:
        G = capi.Engine(V_dim=10, **FIXED, V_capacity=512, V_capacity_max=M, **kw)
        F = capi.Engine(V_dim=10, **FIXED, V_capacity=M, **kw)
    want = []
    for t, b in enumerate(batches):
        rg, pg = raw_rc(G, b)
        rf, pf = raw_rc(F, b)
        assert rg == rf, (t, rg, rf, G.L.dfb_last_error(G.h).decode())
        want.append(rg)
        if rg == 0:
            assert pg == pf, t
    assert want[3] == capi.DFB_ERR_CAPACITY and want[:3] == [0, 0, 0], want
    for x, y in zip(G.read_entries(idr.seen_keys(batches)), F.read_entries(idr.seen_keys(batches))):
        assert np.array_equal(x, y)
    assert G.table_stats() == F.table_stats() and G.rng_state() == F.rng_state()


def trained_model(V_dim=16, nb=5):
    rng = np.random.default_rng(23)
    A = capi.Engine(V_dim=V_dim, **FIXED, **KW)
    for b in batches_of(rng, False)[:nb]:
        A.train_step_raw(b[0], b[2], b[3], b[1], True, True)
    return A


def test_restore_beyond_the_initial_capacity():
    A = trained_model()
    blob = A.snapshot()
    assert A.table_stats()["n_keys"] > 4 * 1024
    G, T = twins(16)
    G.restore_from(io.BytesIO(blob), chunk_bytes=4096)
    T.restore_from(io.BytesIO(blob), chunk_bytes=4096)
    assert G.snapshot() == blob == T.snapshot()
    # and the restored engines train alike
    b = batches_of(np.random.default_rng(5), True)[4]
    assert idr.as_tuple(G.train_step_raw(b[0], b[2], b[3], b[1])) == idr.as_tuple(T.train_step_raw(b[0], b[2], b[3], b[1]))
    assert_same_end(G, T)


def test_restore_two_parts_into_three_growing_ranks():
    from test_gpu_checkpoint import restore_parts
    A = trained_model()
    blob = A.snapshot()
    parts = []
    for r in range(2):                  # the model as two ranks of a 2-GPU run would have saved it
        P = capi.Engine(V_dim=16, **FIXED, **KW)
        P.restore_from(io.BytesIO(blob), shard=r, nshards=2)
        parts.append(P.snapshot())
    grow = [capi.Engine(V_dim=16, **GROW, **KW) for _ in range(3)]
    fixed = [capi.Engine(V_dim=16, **FIXED, **KW) for _ in range(3)]
    restore_parts(grow, parts)
    restore_parts(fixed, parts)
    for g, f in zip(grow, fixed):
        assert g.snapshot() == f.snapshot() and g.rng_state() == f.rng_state()
    assert sum(g.table_stats()["n_keys"] for g in grow) == A.table_stats()["n_keys"]
    assert max(g.table_stats()["capacity"] for g in grow) > 1024


def test_replaced_tables_are_freed():
    """after growing to about 2 M keys, the device has as much free memory as with a pre-sized engine of the same final
    capacities (slack: 64 MiB for allocation rounding; the last table replaced alone holds 128 MiB)"""
    rng = np.random.default_rng(29)
    batches = [tlf.big_batch(rng, np.unique(rng.integers(0, 1 << 40, 1 << 21).astype(U64) * GOLDEN), 20000 * (j + 1),
                             False) for j in range(3)]

    def free_after(E):
        for b in batches:
            E.train_step_raw(b[0], b[2], b[3], b[1])
        E.sync()
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0], E.table_stats()

    G = capi.Engine(V_dim=16, table_capacity=1024, table_capacity_max=1 << 24, **KW)
    free_g, st = free_after(G)
    G.close()
    assert st["capacity"] > 1 << 21
    P = capi.Engine(V_dim=16, table_capacity=st["capacity"], V_capacity=st["v_capacity"], **KW)
    free_p, st_p = free_after(P)
    assert st_p["capacity"] == st["capacity"]
    assert abs(free_g - free_p) < 64 << 20, (free_g, free_p)


def test_parameter_checks_and_the_sharded_store_refusal():
    for kw in (dict(table_capacity=2048, table_capacity_max=1024), dict(table_capacity_max=(1 << 30) + 1),
               dict(V_capacity=4096, V_capacity_max=2048), dict(V_capacity_max=(1 << 30) + 1)):
        with pytest.raises(capi.DfbError) as e:
            capi.Engine(V_dim=8, **kw)
        assert e.value.code == capi.DFB_ERR_PARAM, kw
    E = capi.Engine(V_dim=8, table_capacity=1024, table_capacity_max=1 << 20)
    with pytest.raises(capi.DfbError) as e:
        E.shard_init(0, 1, 128, 4096)
    assert "does not grow" in str(e.value)
    F = capi.Engine(V_dim=8, table_capacity=1024, table_capacity_max=1024)    # at its maximum: a fixed engine
    F.shard_init(0, 1, 128, 4096)


def test_cli_trains_from_a_small_table(tmp_path):
    from test_gpu_checkpoint import write_libsvm
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    exe = os.path.join(hb.build(), "difacto_b200")
    data = str(tmp_path / "d.libsvm")
    write_libsvm(data, 3000, 6)
    assert len(set(kv.split(":")[0] for line in open(data) for kv in line.split()[1:])) > 1024
    conf = ["V_dim=16", "l1=0.05", "l2=0.01", "lr=0.2", "V_lr=0.1", "V_threshold=1", "V_l2=0.01", "V_init_scale=0.2",
            "seed=3", "batch_size=200", "max_num_epochs=2", "stop_rel_objv=0", "num_gpus=1"]

    def run(extra, model):
        out = subprocess.run([exe, f"data_in={data}", f"model_out={model}"] + conf + extra, capture_output=True,
                             text=True, timeout=300)
        assert out.returncode == 0, out.stderr[-2000:]
        return [ln for ln in out.stdout.splitlines() if "Training:" in ln]

    a = run(["table_capacity=1024", "table_capacity_max=1000000"], tmp_path / "grow")
    b = run(["table_capacity=1000000"], tmp_path / "fixed")
    assert len(a) == 2 and a == b
    assert open(tmp_path / "grow", "rb").read() == open(tmp_path / "fixed", "rb").read()
