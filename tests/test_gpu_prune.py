"""dfb_prune: dropping the entries with w == 0, no V row and fea_cnt <= max_count.

The oracle is exact.  Engine A trains, prunes and trains on.  Its twin B trains identically up to the prune; B's
snapshot, with those records filtered out in Python, is restored into a fresh engine B', which trains on A's batches.
A and B' must agree bitwise: every step's Progress, every predict step's predictions, the final snapshot bytes, the
rand_r state, n_keys and n_vrows; and dfb_prune's count must equal the records filtered out.  (Results do not depend on
where keys and V rows sit: the growth and resume tests rely on that too.)

Covered: V_dim 0, 10 and 64, binary and valued, max_count 0 and positive; an l1 under which most keys keep w = 0, and
l1 = 0 with V_threshold = 0, where far fewer keys qualify, and a second prune that finds nothing and leaves
the snapshot bytes as they were; steps after the prune through the sync, pipelined and
device entry points with push_cnt, validation and predict steps; a lookup-free raw step; predictions right before and
right after a prune; a growing engine against a pre-sized one, and one that fills its freed slots without growing; a fixed engine at its capacity; a frozen copy written
while the engine prunes; 1, 2 and 3 sharded ranks on one GPU; and the CLI's prune_period / prune_count, across a
checkpoint and resume.
"""
import struct
import threading

import numpy as np
import pytest

import test_gpu_id_range as idr
import test_gpu_lookup_free_step as tlf
import test_gpu_table_growth as tg
from shard_sim import make_local, raw_batch, run_local
from test_gpu_resume import Sink, blocking, epoch_lines, exe, run, write_libsvm  # noqa: F401  (exe: the CLI fixture)

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

SPARSE = dict(tg.KW, l1=1.0)                       # most keys keep w = 0
DENSE = dict(tg.KW, l1=0.0, V_threshold=0)         # most keys get w != 0 and a V row
HDR = struct.Struct("<8sIiQQII")


def filtered(blob, c):
    """the snapshot without the records a prune with max_count c drops, and how many it dropped"""
    magic, ver, k, n_keys, n_vrows, seed, aux = HDR.unpack_from(blob, 0)
    fixed = 28 if aux else 20
    row = 4 * k * (2 if aux else 1)
    out, p, dropped = [], HDR.size, 0
    for _ in range(n_keys):
        fea_cnt, w = struct.unpack_from("<ff", blob, p + 8)
        (has_v,) = struct.unpack_from("<i", blob, p + fixed - 4)
        n = fixed + (row if has_v else 0)
        if w == 0 and has_v == 0 and fea_cnt <= c:
            dropped += 1
        else:
            out.append(blob[p:p + n])
        p += n
    assert p == len(blob)
    return HDR.pack(magic, ver, k, n_keys - dropped, n_vrows, seed, aux) + b"".join(out), dropped


def restored(B, c, **kw):
    """B' of the module docstring: a fresh engine holding B's filtered model, with B's id range"""
    blob, dropped = filtered(B.snapshot(), c)
    Bp = capi.Engine(**kw)
    Bp.restore(blob)
    if B.id_range():
        Bp.set_id_range(B.id_range())
    return Bp, dropped


BEFORE = [("train", 0, True), ("train", 1, False), ("val", 2, False), ("train", 2, False)]
AFTER = [("train", 2, False), ("predict", 3, False), ("train", 3, True), ("val", 1, False), ("train", 4, False),
         ("predict", 4, False), ("train", 0, False), ("predict", 1, False)]


def prune_case(V_dim, valued, c, kw, entry, seed):
    rng = np.random.default_rng(seed)
    batches = tg.batches_of(rng, valued)
    ekw = dict(V_dim=V_dim, **tg.FIXED, **kw)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    pa, _ = tg.run_steps(A, batches, BEFORE, entry)
    pb, _ = tg.run_steps(B, batches, BEFORE, "sync")
    assert pa == pb
    o, l, i, v = batches[3]
    _, q0 = A.predict_raw(o, i, v, l)
    before = A.table_stats()
    n = A.prune(c)
    _, q1 = A.predict_raw(o, i, v, l)
    assert np.array_equal(q0, q1), "a prune changes no prediction"
    after = A.table_stats()
    assert after["n_keys"] == before["n_keys"] - n and after["n_vrows"] == before["n_vrows"]
    assert after["capacity"] == before["capacity"]
    Bp, dropped = restored(B, c, **ekw)
    assert n == dropped
    pa, qa = tg.run_steps(A, batches, AFTER, entry)
    pb, qb = tg.run_steps(Bp, batches, AFTER, "sync")
    assert pa == pb
    assert len(qa) == 3 and all(np.array_equal(x, y) for x, y in zip(qa, qb))
    tg.assert_same_end(A, Bp)
    return n, before["n_keys"]


@pytest.mark.parametrize("entry", ["sync", "async", "dev"])
@pytest.mark.parametrize("V_dim,valued,c", [(0, False, 0.0), (10, True, 2.0), (64, False, 0.0), (64, True, 3.0)])
def test_prune_equals_a_restore_of_the_filtered_snapshot(entry, V_dim, valued, c):
    n, keys = prune_case(V_dim, valued, c, SPARSE, entry, 5 * V_dim + valued)
    assert n > keys // 3, (n, keys)               # l1 = 1: much of the table goes


@pytest.mark.parametrize("V_dim,valued,c", [(10, False, 0.0), (64, True, 5.0)])
def test_prune_where_few_keys_qualify(V_dim, valued, c):
    rng = np.random.default_rng(61 + V_dim)
    batches = tg.batches_of(rng, valued)
    ekw = dict(V_dim=V_dim, **tg.FIXED, **DENSE)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    assert tg.run_steps(A, batches, BEFORE, "sync") == tg.run_steps(B, batches, BEFORE, "sync")
    blob = A.snapshot()
    n = A.prune(c)
    assert n == filtered(blob, c)[1]
    # nothing qualifies: the table is left as it was
    blob = A.snapshot()
    assert A.prune(c) == 0 and A.prune(-1.0) == 0 and A.snapshot() == blob
    Bp, _ = restored(B, c, **ekw)
    pa, qa = tg.run_steps(A, batches, AFTER, "sync")
    pb, qb = tg.run_steps(Bp, batches, AFTER, "sync")
    assert pa == pb and all(np.array_equal(x, y) for x, y in zip(qa, qb))
    tg.assert_same_end(A, Bp)


def test_lookup_free_step_after_a_prune():
    rng = np.random.default_rng(43)
    pool = np.unique(rng.integers(0, 1 << 40, 700000).astype(tg.U64) * tg.GOLDEN)
    batches = [tlf.big_batch(rng, pool[:400000], 70000, False, pool[3]),
               tlf.big_batch(rng, pool[200000:], 70000, True, pool[3])]
    assert tlf.above_l2_bound(batches)
    ekw = dict(V_dim=16, table_capacity=1 << 21, **SPARSE)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    plan = [("train", 0, True)]
    assert tg.run_steps(A, batches, plan, "sync") == tg.run_steps(B, batches, plan, "sync")
    n = A.prune(1.0)
    Bp, dropped = restored(B, 1.0, **ekw)
    assert n == dropped > 0
    plan = [("train", 1, False), ("predict", 0, False), ("train", 0, False)]
    pa, qa = tg.run_steps(A, batches, plan, "async")
    pb, qb = tg.run_steps(Bp, batches, plan, "sync")
    assert pa == pb and np.array_equal(qa[0], qb[0])
    tg.assert_same_end(A, Bp)
    tlf.assert_ran_without_lookup(A, batches[1])


def test_growing_engine_pruned_mid_run_then_grown_again():
    rng = np.random.default_rng(47)
    batches = tg.batches_of(rng, True)
    G = capi.Engine(V_dim=10, **tg.GROW, **SPARSE)
    T = capi.Engine(V_dim=10, **tg.FIXED, **SPARSE)
    assert tg.run_steps(G, batches, BEFORE, "async") == tg.run_steps(T, batches, BEFORE, "sync")
    cap0 = G.table_stats()["capacity"]
    n = G.prune(1.0)
    assert n == T.prune(1.0) > 0
    assert G.table_stats()["capacity"] == cap0
    caps = []
    pg, qg = tg.run_steps(G, batches, AFTER, "async", caps)
    pt, qt = tg.run_steps(T, batches, AFTER, "sync")
    assert pg == pt and all(np.array_equal(x, y) for x, y in zip(qg, qt))
    assert max(c[0] for c in caps) > cap0, "the table must grow again after the prune"
    tg.assert_same_end(G, T)


def test_a_growing_engine_reuses_the_freed_slots():
    """after a prune the growth bookkeeping knows the table's real count: a batch of b new keys with
    n_keys after the prune + b <= capacity < n_keys before it + b fits without growing"""
    rng = np.random.default_rng(67)
    batches = tg.batches_of(rng, False)
    G = capi.Engine(V_dim=10, table_capacity=1024, table_capacity_max=1 << 22, **SPARSE)
    tg.run_steps(G, batches, BEFORE, "sync")
    st = G.table_stats()
    cap, K = st["capacity"], st["n_keys"]
    D = G.prune(1.0)
    b = cap - (K - D)
    assert D > 0 and b > cap - K
    ids = np.unique(rng.integers(1 << 41, 1 << 42, 2 * b).astype(tg.U64) * tg.GOLDEN)[:b]
    rng.shuffle(ids)
    assert len(ids) == b
    lens = np.full(b // 20, 20)
    if b % 20:
        lens = np.append(lens, b % 20)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(tg.U64)
    lab = np.where(rng.random(len(lens)) < 0.4, 1.0, -1.0).astype(np.float32)
    G.train_step_raw(off, ids, None, lab, False, True)
    st = G.table_stats()
    assert st["capacity"] == cap, "the table grew although the freed slots held the batch"
    assert st["n_keys"] == cap


def test_a_prune_makes_room_in_a_fixed_table():
    rng = np.random.default_rng(53)
    batches = tg.batches_of(rng, False)
    ekw = dict(V_dim=10, **SPARSE)
    R = capi.Engine(table_capacity=1 << 18, **ekw)        # the counts without a limit
    P = capi.Engine(table_capacity=1 << 18, **ekw)        # and with the prune before step 3
    for t in range(3):
        assert tg.raw_rc(R, batches[t])[0] == 0 and tg.raw_rc(P, batches[t])[0] == 0
    k2 = R.table_stats()["n_keys"]
    assert P.prune(1.0) > 0
    assert tg.raw_rc(R, batches[3])[0] == 0 and tg.raw_rc(P, batches[3])[0] == 0
    k3, k3p = R.table_stats()["n_keys"], P.table_stats()["n_keys"]
    M = max(k2, k3p)
    assert M < k3
    F, Fp = capi.Engine(table_capacity=M, **ekw), capi.Engine(table_capacity=M, **ekw)
    for t in range(3):
        assert tg.raw_rc(F, batches[t])[0] == 0 and tg.raw_rc(Fp, batches[t])[0] == 0
    Fp.prune(1.0)
    assert tg.raw_rc(F, batches[3])[0] == capi.DFB_ERR_CAPACITY
    rc, pr = tg.raw_rc(Fp, batches[3])
    assert rc == 0 and Fp.table_stats()["n_keys"] == k3p
    assert Fp.snapshot() == P.snapshot()


def test_a_frozen_copy_is_not_changed_by_a_prune():
    rng = np.random.default_rng(59)
    batches = tg.batches_of(rng, True)
    A = capi.Engine(V_dim=16, **tg.FIXED, **SPARSE)
    tg.run_steps(A, batches, BEFORE, "sync")
    want = blocking(A)
    f = A.snapshot_begin()
    sink, err = Sink(), []

    def write():
        try:
            f.write_to(sink, chunk_bytes=4096)
        except Exception as e:          # surfaced below
            err.append(e)
    th = threading.Thread(target=write)
    th.start()
    assert A.prune(2.0) > 0
    th.join()
    assert not err, err
    assert sink.value() == want
    again = Sink()
    f.write_to(again)
    assert again.value() == want and blocking(A) != want
    f.release()


@pytest.mark.parametrize("S", [1, 2, 3])
def test_sharded_ranks_prune_between_steps(S):
    kw = dict(SPARSE, V_dim=16)
    kw.pop("id_bits")
    fn = lambda r, s: raw_batch(r, s, s % 2 == 0, B=120, ids=3000, seed=13)   # noqa: E731
    A, pa = run_local(S, kw, 4, fn)
    B, pb = run_local(S, kw, 4, fn)
    assert [[idr.as_tuple(p) for p in x] for x in pa] == [[idr.as_tuple(p) for p in x] for x in pb]
    # not during a step
    for E in A:
        off, idx, val, lab = fn(0, 9)
        E.shard_begin_async(len(lab), off, idx, val, lab, push_cnt=False, is_train=False)
    with pytest.raises(capi.DfbError) as e:
        A[0].prune(1.0)
    assert e.value.code == capi.DFB_ERR_INVALID
    for phase in range(5):
        for E in A:
            E.shard_phase(phase)
    for E in A:
        E.wait_step()
    for E in B:       # the twin takes the same validation step
        off, idx, val, lab = fn(0, 9)
        E.shard_begin_async(len(lab), off, idx, val, lab, push_cnt=False, is_train=False)
    for phase in range(5):
        for E in B:
            E.shard_phase(phase)
    for E in B:
        E.wait_step()
    Bp = make_local(S, kw)
    total = 0
    for r in range(S):
        blob, dropped = filtered(B[r].snapshot(), 1.0)
        Bp[r].restore(blob)
        n = A[r].prune(1.0)
        assert n == dropped, f"rank {r}"
        total += n
    assert total > 0
    g = lambda r, s: fn(r, s + 4)   # noqa: E731
    _, pa = run_local(S, kw, 4, g, engines=A, cnt_steps=1)
    _, pb = run_local(S, kw, 4, g, engines=Bp, cnt_steps=1)
    assert [[idr.as_tuple(p) for p in x] for x in pa] == [[idr.as_tuple(p) for p in x] for x in pb]
    for r in range(S):
        tg.assert_same_end(A[r], Bp[r])


# ---------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------
def prune_lines(out):
    return [ln for ln in out.split("\n") if ln.startswith("Prune: ")]


def cli_case(exe, tmp_path, num_gpus):   # noqa: F811
    data, val = str(tmp_path / "train.libsvm"), str(tmp_path / "val.libsvm")
    write_libsvm(data, 1500, 3)
    write_libsvm(val, 300, 4)
    common = [f"data_in={data}", f"data_val={val}", "V_dim=16", "l1=1", "lr=0.2", "V_threshold=2", "batch_size=50",
              "shuffle=2", "num_jobs_per_epoch=3", "stop_rel_objv=0", "stop_val_auc=-2", "table_capacity=65536", f"num_gpus={num_gpus}",
              "prune_period=5", "prune_count=2"]
    C_ = run(exe, common + ["max_num_epochs=3", f"model_out={tmp_path / 'c.model'}"])
    assert C_.returncode == 0, C_.stderr[-2000:]
    lines = prune_lines(C_.stdout)
    assert len(lines) >= 5 and sum(int(ln.split("dropped ")[1].split(",")[0]) for ln in lines) > 0, lines
    P = str(tmp_path / "ckpt")
    # 30 minibatches per epoch: the last checkpoint of 2 epochs is at minibatch 35, mid-part and on a prune boundary,
    # where the prune runs first and the checkpoint holds the pruned model
    A = run(exe, common + ["max_num_epochs=2", f"checkpoint_out={P}", "checkpoint_period=35"])
    assert A.returncode == 0, A.stderr[-2000:]
    assert prune_lines(A.stdout) == lines[:len(prune_lines(A.stdout))]
    B = run(exe, common + ["max_num_epochs=3", f"checkpoint_in={P}", f"model_out={tmp_path / 'b.model'}"])
    assert B.returncode == 0, B.stderr[-2000:]
    head = B.stdout.split("Resuming from checkpoint")[1].split("\n")[0]
    epoch, m = int(head.split("epoch ")[1].split(",")[0]), int(head.split("minibatch ")[1])
    assert m % 5 == 0 and any(ln.startswith(f"Prune: minibatch {m},") for ln in lines)
    assert epoch_lines(B.stdout, epoch) == epoch_lines(C_.stdout, epoch)
    after = [ln for ln in lines if int(ln.split("minibatch ")[1].split(",")[0]) > m]
    assert after and prune_lines(B.stdout) == after, "the prunes after the checkpoint"
    for r in range(num_gpus):
        name = (lambda b: f"{b}_part-{r}") if num_gpus > 1 else (lambda b: b)
        assert open(name(tmp_path / "b.model"), "rb").read() == open(name(tmp_path / "c.model"), "rb").read()
    bad = run(exe, [a for a in common if not a.startswith("prune_count")] + ["prune_count=3", f"checkpoint_in={P}"])
    assert bad.returncode != 0 and "prune_count" in bad.stderr


def test_cli_prune_one_gpu(exe, tmp_path):   # noqa: F811
    cli_case(exe, tmp_path, 1)


def test_cli_prune_two_gpus(exe, tmp_path):   # noqa: F811
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cli_case(exe, tmp_path, 2)


def test_prune_arguments():
    E = capi.Engine(V_dim=4, table_capacity=1024)
    assert E.prune() == 0
    with pytest.raises(capi.DfbError) as e:
        E.prune(float("nan"))
    assert e.value.code == capi.DFB_ERR_INVALID
    assert E.table_stats()["n_keys"] == 0
