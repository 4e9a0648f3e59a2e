"""Growing ranks of the fused sharded store (shard_growth = 1) against pre-sized twins.

Every test runs S ranks in one process on one GPU (tests/shard_sim.py) that start from table_capacity = 1024 and a
small V_capacity, on batches that bring new keys every step, and a twin store of ranks pre-sized for the whole run.
Growth moves every key to another slot, so equality here is bit for bit: Progress, every entry, the InitV stream,
predictions."""
import gc
import io
import os
import subprocess
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from difacto_b200.sharded import FusedShardedStore  # noqa: E402
from shard_sim import all_keys, enqueue_local, key_owner_np, make_local, raw_batch  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=0, V_l2=0.01, V_init_scale=0.2, seed=3)
GROW = dict(table_capacity=1024, V_capacity=256, table_capacity_max=1 << 20, V_capacity_max=1 << 20, shard_growth=1)
FIXED = dict(table_capacity=1 << 18, V_capacity=1 << 18)
SHARD = dict(max_rows=512, max_nnz=1 << 17)
STEPS, CNT_STEPS = 8, 6
GRANULE = 2 << 20      # the VMM allocation granularity the V-row pool is mapped in (2 MiB on the H100)


def fn_of(seed, B=400, ids=1 << 30, max_nnz=48):
    """step s, rank r: a batch of B rows over `ids` ids (new keys every step), binary on odd steps"""
    return lambda r, s: raw_batch(r, s, s % 2 == 0, B=B, ids=ids, max_nnz=max_nnz, seed=seed)


@pytest.fixture(autouse=True)
def release_engines():
    """the engines of a test (a frozen copy refers back to its engine) are gone before the next test measures memory"""
    yield
    gc.collect()
    torch.cuda.synchronize()


def progress(p):
    return tuple(p.as_dict().values())


def step_all(engines, batches, push_cnt, is_train):
    """one step of every rank; each rank's Progress, or the error code its wait reports"""
    enqueue_local(engines, batches, push_cnt, is_train)
    out = []
    for E in engines:
        try:
            out.append(progress(E.wait_step()))
        except capi.DfbError as e:
            out.append(("error", e.code))
    return out


def received(batches, S):
    """the keys each owner receives in one step: the unique keys of every worker's batch that fall into its range"""
    n = np.zeros(S, np.int64)
    for off, idx, _, _ in batches:
        own = key_owner_np(np.unique(idx), S)
        n += np.bincount(own, minlength=S)
    return n


def make(S, V_dim, engine_kw, kw=KW, **shard_kw):
    return make_local(S, dict(kw, V_dim=V_dim), engine_kw=engine_kw, **dict(SHARD, **shard_kw))


def assert_same_model(A, B, keys, S):
    own = key_owner_np(keys, S)
    for s in range(S):
        for x, y in zip(A[s].read_entries(keys[own == s]), B[s].read_entries(keys[own == s])):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), f"rank {s}"
        assert A[s].rng_state() == B[s].rng_state(), f"rank {s}"
        a, b = A[s].table_stats(), B[s].table_stats()
        assert (a["n_keys"], a["n_vrows"]) == (b["n_keys"], b["n_vrows"]), f"rank {s}"


@pytest.mark.parametrize("V_dim", [0, 10, 64])
@pytest.mark.parametrize("S", [1, 2, 3])
def test_growing_ranks_equal_presized_ranks(S, V_dim):
    fn = fn_of(S * 100 + V_dim)
    G = make(S, V_dim, GROW)
    T = make(S, V_dim, FIXED)
    caps = [[] for _ in range(S)]
    Kseg = G[0].shard_info()["seg_keys"]
    for t in range(STEPS):
        batches = [fn(r, t) for r in range(S)]
        before = [E.table_stats() for E in G]
        pg = step_all(G, batches, t < CNT_STEPS, True)
        pt = step_all(T, batches, t < CNT_STEPS, True)
        assert pg == pt, f"step {t}"
        rcv = received(batches, S)
        for r, E in enumerate(G):
            st = E.table_stats()
            caps[r].append((st["capacity"], st["v_capacity"]))
            if st["capacity"] != before[r]["capacity"]:
                assert st["capacity"] < 2 * (st["n_keys"] + rcv[r]), (t, r, st, rcv[r])
            if st["v_capacity"] != before[r]["v_capacity"]:
                slack = GRANULE // E.row_bytes()[0]
                assert st["v_capacity"] < 2 * (st["n_vrows"] + rcv[r]) + slack, (t, r, st, rcv[r])
        # far below the worst case the host would otherwise have had to reserve for: S segments of seg_keys keys
        assert 8 * int(rcv.max()) < S * Kseg
    assert_same_model(G, T, all_keys(S, STEPS, fn), S)
    assert max(len(set(c[0] for c in cr)) for cr in caps) >= 3, caps
    if V_dim:
        assert max(len(set(c[1] for c in cr)) for cr in caps) >= 3, caps


def test_validation_and_predict_steps_do_not_grow():
    S, V_dim = 2, 16
    fn = fn_of(7)
    G, T = make(S, V_dim, GROW), make(S, V_dim, FIXED)
    for t in range(6):
        batches = [fn(r, t) for r in range(S)]
        assert step_all(G, batches, t < 2, True) == step_all(T, batches, t < 2, True)
        caps = [E.table_stats() for E in G]
        new = [fn(r, 50 + t) for r in range(S)]          # keys the model has not seen
        assert step_all(G, new, False, False) == step_all(T, new, False, False)
        preds = []
        for engines in (G, T):
            out = [np.zeros(len(b[3]), np.float32) for b in new]
            for E, (off, idx, val, lab), o in zip(engines, new, out):
                E.shard_begin_predict_async(len(lab), off, idx, val, lab, o)
            for phase in range(5):
                for E in engines:
                    E.shard_phase(phase)
            for E in engines:
                E.wait_step()
            preds.append(out)
        for a, b in zip(*preds):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert [E.table_stats() for E in G] == caps
    assert_same_model(G, T, all_keys(S, 6, fn), S)


def test_dropped_batches_behave_as_on_the_twin():
    """a worker's segment over seg_keys, and a batch with an id outside id_bits, are dropped on both stores alike"""
    S, V_dim = 2, 10
    base = fn_of(11, B=200, max_nnz=24)

    def fn(r, s):
        off, idx, val, lab = base(r, s)
        idx = idx >> np.uint64(24)                      # ids below 2^40
        if s == 2 and r == 0:                           # a larger batch: its segments exceed seg_keys
            off, idx, val, lab = raw_batch(r, 90, val is not None, B=500, ids=1 << 30, max_nnz=24, seed=11)
            idx = idx >> np.uint64(24)
        if s == 4 and r == 1:
            idx = idx.copy()
            idx[len(idx) // 2] = np.uint64(1 << 45)     # out of range
        return off, idx, val, lab

    kw = dict(KW, id_bits=40)
    G = make(S, V_dim, GROW, kw=kw, seg_keys=2000)
    T = make(S, V_dim, FIXED, kw=kw, seg_keys=2000)
    codes = set()
    for t in range(6):
        batches = [fn(r, t) for r in range(S)]
        pg, pt = step_all(G, batches, t < 3, True), step_all(T, batches, t < 3, True)
        assert pg == pt, f"step {t}"
        codes |= {p[1] for p in pg if p[0] == "error"}
    assert codes, "no batch was dropped"
    assert_same_model(G, T, all_keys(S, 6, fn), S)


@pytest.mark.parametrize("which", ["table", "V"])
def test_the_maximum_reports_capacity_like_a_presized_store(which):
    S, V_dim = 2, 10
    fn = fn_of(13)
    cap = 6000
    if which == "table":
        grow = dict(GROW, table_capacity_max=cap)
        fixed = dict(table_capacity=cap, V_capacity=1 << 18)
    else:
        grow = dict(GROW, V_capacity_max=cap)
        fixed = dict(table_capacity=1 << 18, V_capacity=cap)
    G, T = make(S, V_dim, grow), make(S, V_dim, fixed)
    # which keys of the overflowing step still got in depends on thread order, on either store: compare up to it
    for t in range(STEPS):
        batches = [fn(r, t) for r in range(S)]
        pg, pt = step_all(G, batches, True, True), step_all(T, batches, True, True)
        err_g = [p if p[0] == "error" else None for p in pg]
        assert err_g == [p if p[0] == "error" else None for p in pt], f"step {t}"
        if any(err_g):
            assert ("error", capi.DFB_ERR_CAPACITY) in err_g
            break
        assert pg == pt, f"step {t}"
    else:
        raise AssertionError("the maximum was never reached")


def test_prune_mid_run_then_grow_again():
    S, V_dim = 2, 10
    fn = fn_of(17)
    G, T = make(S, V_dim, GROW), make(S, V_dim, FIXED)
    for t in range(8):
        batches = [fn(r, t) for r in range(S)]
        assert step_all(G, batches, t < 2, True) == step_all(T, batches, t < 2, True), f"step {t}"
        if t == 3:
            dropped = [E.prune(1.0) for E in G]
            assert dropped == [E.prune(1.0) for E in T]
            assert sum(dropped) > 0
    for g, f in zip(G, T):
        assert g.snapshot() == f.snapshot() and g.rng_state() == f.rng_state()


def test_frozen_parts_of_growing_ranks_restore_into_three_growing_ranks():
    from test_gpu_checkpoint import restore_parts
    S, V_dim = 2, 16
    fn = fn_of(19)
    G, T = make(S, V_dim, GROW), make(S, V_dim, FIXED)
    for t in range(4):
        batches = [fn(r, t) for r in range(S)]
        assert step_all(G, batches, t < 2, True) == step_all(T, batches, t < 2, True)
    frozen = [E.snapshot_begin() for E in G]
    want = [E.snapshot() for E in T]
    for t in range(4, 6):                               # the growing ranks keep training and growing meanwhile
        batches = [fn(r, t) for r in range(S)]
        assert step_all(G, batches, False, True) == step_all(T, batches, False, True)
    parts = []
    for f in frozen:
        buf = io.BytesIO()
        f.write_to(buf, chunk_bytes=4096)
        f.release()
        parts.append(buf.getvalue())
    assert parts == want
    ranks = []
    for ekw in (GROW, FIXED):
        engines = [capi.Engine(V_dim=V_dim, **KW, **ekw) for _ in range(3)]
        restore_parts(engines, parts)
        FusedShardedStore.connect_local(engines, **SHARD)
        ranks.append(engines)
    g3 = lambda r, s: fn(r, s + 10)                   # noqa: E731
    for t in range(5):
        batches = [g3(r, t) for r in range(3)]
        assert step_all(ranks[0], batches, t < 1, True) == step_all(ranks[1], batches, t < 1, True), f"step {t}"
    for g, f in zip(*ranks):
        assert g.snapshot() == f.snapshot() and g.rng_state() == f.rng_state()


def test_one_thread_per_rank():
    """each rank driven by its own host thread (dfb_shard_step_async enqueues all five phases of one rank), so a rank's
    blocking wait for its step's count may come before another rank has enqueued its phase 0 of that step"""
    import threading
    S, V_dim = 3, 16
    fn = fn_of(29)
    G, T = make(S, V_dim, GROW), make(S, V_dim, FIXED)
    prog, errors = [[] for _ in range(S)], []

    def drive(r):
        try:
            for t in range(STEPS):
                off, idx, val, lab = fn(r, t)
                G[r].shard_step_async(len(lab), off, idx, val, lab, push_cnt=t < CNT_STEPS, is_train=True)
                prog[r].append(progress(G[r].wait_step()))
        except Exception as e:      # noqa: BLE001 -- reported below
            errors.append((r, e))

    th = [threading.Thread(target=drive, args=(r,)) for r in range(S)]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=300)
    assert not any(x.is_alive() for x in th), "a rank's thread did not finish"
    assert not errors, errors
    for t in range(STEPS):
        assert step_all(T, [fn(r, t) for r in range(S)], t < CNT_STEPS, True) == [prog[r][t] for r in range(S)], t
    assert_same_model(G, T, all_keys(S, STEPS, fn), S)
    assert sum(E.growth_stats()[0] for E in G) >= 3


def _ipc_worker(rank, world, port, out, grow):
    """one rank per process and GPU, connected over CUDA IPC; every rank calls dfb_shard_step_async"""
    import torch.distributed as dist
    from difacto_b200 import capi as C2
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    fn = fn_of(31)
    E = C2.Engine(device=rank, V_dim=16, **KW, **(GROW if grow else FIXED))
    FusedShardedStore(E, **SHARD)
    prog = []
    for t in range(STEPS):
        off, idx, val, lab = fn(rank, t)
        E.shard_step_async(len(lab), off, idx, val, lab, push_cnt=t < CNT_STEPS, is_train=True)
        prog.append(progress(E.wait_step()))
    keys = all_keys(world, STEPS, fn)
    scal, hasv, V, cg = E.read_entries(keys[key_owner_np(keys, world) == rank])
    st = E.table_stats()
    np.savez(out.format(rank=rank), scal=scal, hasv=hasv, V=V, cg=cg, prog=np.array(prog, dtype=np.float64),
             rng=E.rng_state(), counts=np.array([st["n_keys"], st["n_vrows"]]), growths=E.growth_stats()[0])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_ipc_one_process_per_rank(tmp_path):
    import socket
    import torch.multiprocessing as mp
    world = 2
    res = {}
    for grow in (True, False):
        sk = socket.socket()
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
        sk.close()
        out = str(tmp_path / f"grow{int(grow)}_{{rank}}.npz")
        mp.spawn(_ipc_worker, args=(world, port, out, grow), nprocs=world, join=True)
        res[grow] = [np.load(out.format(rank=r)) for r in range(world)]
    for r in range(world):
        g, f = res[True][r], res[False][r]
        for k in ("scal", "hasv", "V", "cg", "prog", "rng", "counts"):
            assert np.array_equal(np.asarray(g[k]).view(np.uint8), np.asarray(f[k]).view(np.uint8)), (r, k)
    assert sum(int(res[True][r]["growths"]) for r in range(world)) >= 2


def test_keys_and_refusals():
    E = capi.Engine(V_dim=8, table_capacity=1024, table_capacity_max=1 << 20, shard_growth=0)
    with pytest.raises(capi.DfbError) as e:
        E.shard_init(0, 1, 128, 4096)
    assert e.value.code == capi.DFB_ERR_INVALID and "does not grow" in str(e.value)
    with pytest.raises(capi.DfbError) as e:
        capi.Engine(V_dim=8, shard_growth=2)
    assert e.value.code == capi.DFB_ERR_PARAM
    capi.Engine(V_dim=8, table_capacity=1024, table_capacity_max=1 << 20, shard_growth=1).shard_init(0, 1, 128, 4096)


def test_launches_when_nothing_has_to_grow():
    """ample capacity: one count kernel per training step at most; at the maxima: exactly a fixed store's launches"""
    S, V_dim = 2, 16
    fn = fn_of(23)
    # room for the worst case of a step (S x seg_keys = 2^18 keys) beside what the table holds: no growth, no wait
    ample = dict(table_capacity=1 << 19, V_capacity=1 << 19, table_capacity_max=1 << 20, V_capacity_max=1 << 20,
                 shard_growth=1)
    at_max = dict(FIXED, shard_growth=1)
    stores = [make(S, V_dim, ekw) for ekw in (FIXED, ample, at_max)]
    for t in range(4):
        batches = [fn(r, t) for r in range(S)]
        counts = []
        for engines in stores:
            c0 = [E.launch_count() for E in engines]
            step_all(engines, batches, t < 2, True)
            counts.append([E.launch_count() - c for E, c in zip(engines, c0)])
        fixed, grow, maxed = counts
        assert maxed == fixed, t
        assert all(g - f in (0, 1) for g, f in zip(grow, fixed)), (t, grow, fixed)
    assert [E.growth_stats() for E in stores[1]] == [(0, 0)] * S


def test_cli_two_gpus_from_a_small_table(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from test_gpu_checkpoint import write_libsvm
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    exe = os.path.join(hb.build(), "difacto_b200")
    data = str(tmp_path / "d.libsvm")
    write_libsvm(data, 3000, 6)
    conf = ["V_dim=16", "l1=0.05", "l2=0.01", "lr=0.2", "V_lr=0.1", "V_threshold=1", "V_l2=0.01", "V_init_scale=0.2",
            "seed=3", "batch_size=200", "max_num_epochs=2", "stop_rel_objv=0", "num_gpus=2"]

    def run(extra, model):
        out = subprocess.run([exe, f"data_in={data}", f"model_out={model}"] + conf + extra, capture_output=True,
                             text=True, timeout=300)
        assert out.returncode == 0, out.stderr[-2000:]
        return [ln for ln in out.stdout.splitlines() if "Training:" in ln]

    a = run(["shard_growth=1", "table_capacity=1024", "table_capacity_max=1000000"], tmp_path / "grow")
    b = run(["table_capacity=1000000"], tmp_path / "fixed")
    assert len(a) == 2 and a == b
    for r in range(2):
        assert open(f"{tmp_path / 'grow'}_part-{r}", "rb").read() == open(f"{tmp_path / 'fixed'}_part-{r}", "rb").read()
