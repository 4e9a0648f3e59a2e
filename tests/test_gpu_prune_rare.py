"""dfb_prune_rare: dropping every entry with fea_cnt <= max_count, V rows included, and compacting the V-row pool.

The oracle is the one of test_gpu_prune.py, with the filter widened.  Engine A trains, prunes and trains on.  Its twin B
trains identically up to the prune; B's snapshot, without the records of fea_cnt <= c and with both header counts
lowered, is restored into a fresh engine B', which lays its rows out in key order and trains on A's batches.  A and B'
must agree bitwise: every step's Progress, every predict step's predictions, the final snapshot bytes with aux data,
the rand_r state, n_keys, n_vrows and the row pool's bytes in use; and the call's counts must equal the records
filtered out and those of them with a V row.  The batches after the prune revisit the kept keys, so two kept keys
sharing a row, or a row copied short, shows in the snapshot.

Covered: V_dim 0, 10, 64 and 128, binary and valued; DENSE (every counted key with w != 0 gets a row) and SPARSE
settings; max_count values under which no row, some interleaved rows and every kept row move; a second call that
finds nothing; the sync, pipelined, device and lookup-free raw entry points with validation and predict steps; a
growing engine against a pre-sized one; a fixed V-row pool that a stream of new ids outruns many times over under
periodic rare prunes; a frozen copy begun before the prune; 1, 2 and 3 sharded ranks on one GPU; the refusals; and the
CLI's prune_rare across a checkpoint and resume.
"""
import struct
import threading

import numpy as np
import pytest

import test_gpu_id_range as idr
import test_gpu_lookup_free_step as tlf
import test_gpu_table_growth as tg
from shard_sim import make_local, raw_batch, run_local
from test_gpu_prune import DENSE, HDR, SPARSE, prune_lines
from test_gpu_resume import Sink, blocking, epoch_lines, exe, run, write_libsvm  # noqa: F401  (exe: the CLI fixture)

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")


def filtered_rare(blob, c):
    """the snapshot without the records of fea_cnt <= c and with both header counts lowered; (it, records dropped,
    V rows dropped)"""
    magic, ver, k, n_keys, n_vrows, seed, aux = HDR.unpack_from(blob, 0)
    fixed = 28 if aux else 20
    row = 4 * k * (2 if aux else 1)
    out, p, dropped, dropped_v = [], HDR.size, 0, 0
    for _ in range(n_keys):
        (fea_cnt,) = struct.unpack_from("<f", blob, p + 8)
        (has_v,) = struct.unpack_from("<i", blob, p + fixed - 4)
        n = fixed + (row if has_v else 0)
        if fea_cnt <= c:
            dropped += 1
            dropped_v += has_v != 0
        else:
            out.append(blob[p:p + n])
        p += n
    assert p == len(blob)
    return HDR.pack(magic, ver, k, n_keys - dropped, n_vrows - dropped_v, seed, aux) + b"".join(out), dropped, dropped_v


def restored(B, c, **kw):
    """B' of the module docstring; (it, records dropped, V rows dropped)"""
    blob, dropped, dropped_v = filtered_rare(B.snapshot(), c)
    Bp = capi.Engine(**kw)
    Bp.restore(blob)
    if B.id_range():
        Bp.set_id_range(B.id_range())
    return Bp, dropped, dropped_v


def assert_same_end(A, Bp):
    tg.assert_same_end(A, Bp)
    assert A.row_bytes() == Bp.row_bytes()


def prune_and_check(A, B, c, ekw):
    """A.prune_rare(c) against B' of twin B; returns (B', n_dropped, n_vrows_freed)"""
    before = A.table_stats()
    n, nv = A.prune_rare(c)
    after = A.table_stats()
    assert after["n_keys"] == before["n_keys"] - n and after["n_vrows"] == before["n_vrows"] - nv
    assert (after["capacity"], after["v_capacity"]) == (before["capacity"], before["v_capacity"])
    Bp, dropped, dropped_v = restored(B, c, **ekw)
    assert (n, nv) == (dropped, dropped_v)
    return Bp, n, nv


# every training step counts: the keys of each batch collect different counts, and their rows are allocated batch by
# batch, so a threshold drops rows interleaved with the kept ones
BEFORE = [("train", 0, True), ("train", 1, True), ("val", 2, False), ("train", 2, True), ("train", 0, True)]
AFTER = [("train", 2, True), ("predict", 3, False), ("train", 0, True), ("val", 1, False), ("train", 1, True),
         ("predict", 0, False), ("train", 3, True), ("train", 4, False), ("predict", 2, False)]


def rare_case(V_dim, valued, c, kw, entry, seed):
    rng = np.random.default_rng(seed)
    batches = tg.batches_of(rng, valued)
    ekw = dict(V_dim=V_dim, **tg.FIXED, **kw)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    pa, _ = tg.run_steps(A, batches, BEFORE, entry)
    pb, _ = tg.run_steps(B, batches, BEFORE, "sync")
    assert pa == pb
    rows0 = A.table_stats()["n_vrows"]
    Bp, n, nv = prune_and_check(A, B, c, ekw)
    # a second call finds nothing and leaves the model as it is
    blob = A.snapshot()
    assert A.prune_rare(c) == (0, 0) and A.snapshot() == blob
    pa, qa = tg.run_steps(A, batches, AFTER, entry)
    pb, qb = tg.run_steps(Bp, batches, AFTER, "sync")
    assert pa == pb
    assert len(qa) == 3 and all(np.array_equal(x, y) for x, y in zip(qa, qb))
    assert_same_end(A, Bp)
    return n, nv, rows0


@pytest.mark.parametrize("entry", ["sync", "async", "dev"])
@pytest.mark.parametrize("V_dim,valued", [(10, True), (64, False), (128, True)])
def test_rare_prune_with_interleaved_rows(entry, V_dim, valued):
    n, nv, rows = rare_case(V_dim, valued, 2.0, DENSE, entry, 3 * V_dim + valued)
    assert 0 < nv < rows and n >= nv, (n, nv, rows)      # some rows go, among kept ones


@pytest.mark.parametrize("V_dim,valued,c", [(0, False, 2.0), (0, True, 1.0), (64, True, 4.0), (128, False, 3.0)])
def test_rare_prune_sparse(V_dim, valued, c):
    """l1 = 1: most keys keep w = 0 and no row; the few rows belong to keys counted more than V_threshold = 2 times"""
    n, nv, rows = rare_case(V_dim, valued, c, SPARSE, "sync", 11 * V_dim + valued)
    assert n > 0 and nv <= rows and (nv == 0 if V_dim == 0 else rows > 0), (n, nv, rows)


@pytest.mark.parametrize("V_dim", [10, 64])
def test_rare_prune_that_moves_no_row(V_dim):
    """DENSE with V_threshold = 2: the keys of fea_cnt <= 2 have no row, so the rows stay where they are"""
    n, nv, rows = rare_case(V_dim, False, 2.0, dict(DENSE, V_threshold=2), "async", 5 + V_dim)
    assert n > 0 and nv == 0 and rows > 0


def unique_batch(rng, ids, per_row, valued):
    """every id of ids once, per_row to a row"""
    ids = ids.copy()
    rng.shuffle(ids)
    lens = np.full(len(ids) // per_row, per_row)
    if len(ids) % per_row:
        lens = np.append(lens, len(ids) % per_row)
    return idr.csr(rng, lens, ids, valued)


@pytest.mark.parametrize("V_dim,valued", [(16, False), (64, True), (128, False)])
def test_rare_prune_that_moves_every_kept_row(V_dim, valued):
    """2000 keys seen once get rows [0, 2000); 500 keys seen three times get the rows after them.  max_count 1 drops
    the first 2000 with their rows: n_vrows becomes 500 and every kept row moves"""
    rng = np.random.default_rng(71 + V_dim)
    pool = np.unique(rng.integers(0, 1 << 40, 6000).astype(tg.U64) * tg.GOLDEN)
    rng.shuffle(pool)
    once, hot = pool[:2000], pool[2000:2500]
    batches = [unique_batch(rng, once, 20, valued), unique_batch(rng, hot, 10, valued),
               tg.batches_of(rng, valued)[2]]
    ekw = dict(V_dim=V_dim, **tg.FIXED, **DENSE)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    plan = [("train", 0, True), ("train", 1, True), ("train", 1, True), ("train", 1, True)]
    assert tg.run_steps(A, batches, plan, "sync") == tg.run_steps(B, batches, plan, "sync")
    st = A.table_stats()
    assert st["n_keys"] == st["n_vrows"] == 2500
    Bp, n, nv = prune_and_check(A, B, 1.0, ekw)
    assert n == nv == 2000 and A.table_stats()["n_vrows"] == 500
    plan = [("train", 1, True), ("predict", 0, False), ("train", 0, True), ("train", 2, True), ("predict", 1, False)]
    pa, qa = tg.run_steps(A, batches, plan, "dev")
    pb, qb = tg.run_steps(Bp, batches, plan, "sync")
    assert pa == pb and all(np.array_equal(x, y) for x, y in zip(qa, qb))
    assert_same_end(A, Bp)


def test_rare_prune_that_drops_everything():
    rng = np.random.default_rng(83)
    batches = tg.batches_of(rng, True)
    ekw = dict(V_dim=10, **tg.FIXED, **DENSE)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    tg.run_steps(A, batches, BEFORE, "sync")
    tg.run_steps(B, batches, BEFORE, "sync")
    st = A.table_stats()
    assert A.prune_rare(1e30) == (st["n_keys"], st["n_vrows"])
    assert A.table_stats()["n_keys"] == A.table_stats()["n_vrows"] == 0
    Bp, _, _ = restored(B, 1e30, **ekw)
    pa, qa = tg.run_steps(A, batches, AFTER, "sync")
    pb, qb = tg.run_steps(Bp, batches, AFTER, "sync")
    assert pa == pb and all(np.array_equal(x, y) for x, y in zip(qa, qb))
    assert_same_end(A, Bp)


def test_lookup_free_step_after_a_rare_prune():
    rng = np.random.default_rng(43)
    pool = np.unique(rng.integers(0, 1 << 40, 700000).astype(tg.U64) * tg.GOLDEN)
    batches = [tlf.big_batch(rng, pool[:400000], 70000, False, pool[3]),
               tlf.big_batch(rng, pool[200000:], 70000, True, pool[3])]
    assert tlf.above_l2_bound(batches)
    ekw = dict(V_dim=16, table_capacity=1 << 21, **DENSE)
    A, B = capi.Engine(**ekw), capi.Engine(**ekw)
    plan = [("train", 0, True), ("train", 1, True)]
    assert tg.run_steps(A, batches, plan, "sync") == tg.run_steps(B, batches, plan, "sync")
    Bp, n, nv = prune_and_check(A, B, 1.0, ekw)
    assert n >= nv > 0
    plan = [("train", 1, False), ("predict", 0, False), ("train", 0, False)]
    pa, qa = tg.run_steps(A, batches, plan, "async")
    pb, qb = tg.run_steps(Bp, batches, plan, "sync")
    assert pa == pb and np.array_equal(qa[0], qb[0])
    assert_same_end(A, Bp)
    tlf.assert_ran_without_lookup(A, batches[1])


def test_growing_engine_rare_pruned_mid_run():
    rng = np.random.default_rng(47)
    batches = tg.batches_of(rng, True)
    G = capi.Engine(V_dim=10, **tg.GROW, **DENSE)
    T = capi.Engine(V_dim=10, **tg.FIXED, **DENSE)
    assert tg.run_steps(G, batches, BEFORE, "async") == tg.run_steps(T, batches, BEFORE, "sync")
    caps0 = G.table_stats()
    n = G.prune_rare(2.0)
    assert n == T.prune_rare(2.0) and n[1] > 0
    st = G.table_stats()
    assert (st["capacity"], st["v_capacity"]) == (caps0["capacity"], caps0["v_capacity"])
    caps = []
    pg, qg = tg.run_steps(G, batches, AFTER, "async", caps)
    pt, qt = tg.run_steps(T, batches, AFTER, "sync")
    assert pg == pt and all(np.array_equal(x, y) for x, y in zip(qg, qt))
    assert max(c[1] for c in caps) > caps0["v_capacity"], "the pool must grow again after the prune"
    assert_same_end(G, T)


def test_a_fixed_pool_outrun_by_new_ids_under_periodic_rare_prunes():
    """a stream of new ids around a hot set: every batch asks for about 900 new rows of a 2048-row pool, and a rare
    prune after each step frees the rows of the ids seen once, so the pool never fills although far more rows than
    it holds are allocated in all"""
    rng = np.random.default_rng(97)
    V_cap = 2048
    E = capi.Engine(V_dim=16, table_capacity=1 << 14, V_capacity=V_cap, **DENSE)
    hot = np.unique(rng.integers(0, 1 << 40, 400).astype(tg.U64) * tg.GOLDEN)
    total = 0
    for t in range(12):
        fresh = np.unique(rng.integers(1 << 40, 1 << 41, 900).astype(tg.U64) * tg.GOLDEN)
        ids = np.concatenate([fresh, hot[rng.integers(0, len(hot), 900)]])
        b = unique_batch(rng, ids, 18, t % 2 == 1)
        rc, pr = tg.raw_rc(E, b)
        assert rc == 0, (t, E.L.dfb_last_error(E.h).decode())
        total += pr[5]                                  # Progress new_vrows
        n, nv = E.prune_rare(1.0)
        st = E.table_stats()
        assert nv > 0 and st["n_vrows"] <= V_cap and st["v_capacity"] == V_cap, (t, st)
    assert total > 4 * V_cap, total


def test_a_frozen_copy_begun_before_a_rare_prune():
    rng = np.random.default_rng(59)
    batches = tg.batches_of(rng, True)
    A = capi.Engine(V_dim=16, **tg.FIXED, **DENSE)
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
    assert A.prune_rare(2.0)[1] > 0
    th.join()
    assert not err, err
    assert sink.value() == want
    again = Sink()
    f.write_to(again)
    assert again.value() == want and blocking(A) != want
    f.release()


@pytest.mark.parametrize("S", [1, 2, 3])
def test_sharded_ranks_rare_prune_between_steps(S):
    kw = dict(DENSE, V_dim=16)
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
        A[0].prune_rare(1.0)
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
    freed = 0
    for r in range(S):
        blob, dropped, dropped_v = filtered_rare(B[r].snapshot(), 1.0)
        Bp[r].restore(blob)
        assert A[r].prune_rare(1.0) == (dropped, dropped_v), f"rank {r}"
        freed += dropped_v
    assert freed > 0
    g = lambda r, s: fn(r, s + 4)   # noqa: E731
    _, pa = run_local(S, kw, 4, g, engines=A, cnt_steps=1)
    _, pb = run_local(S, kw, 4, g, engines=Bp, cnt_steps=1)
    assert [[idr.as_tuple(p) for p in x] for x in pa] == [[idr.as_tuple(p) for p in x] for x in pb]
    for r in range(S):
        assert_same_end(A[r], Bp[r])


def test_rare_prune_refusals():
    E = capi.Engine(V_dim=4, table_capacity=1024)
    assert E.prune_rare(0.0) == (0, 0)
    with pytest.raises(capi.DfbError) as e:
        E.prune_rare(float("nan"))
    assert e.value.code == capi.DFB_ERR_INVALID
    # a scoring-only engine
    rng = np.random.default_rng(3)
    batches = tg.batches_of(rng, False)
    T = capi.Engine(V_dim=16, **tg.FIXED, **DENSE)
    tg.run_steps(T, batches, BEFORE[:2], "sync")
    S_ = capi.Engine(V_dim=16, **tg.FIXED, **DENSE, score_only=True)
    S_.restore(T.snapshot())
    st = S_.table_stats()
    with pytest.raises(capi.DfbError) as e:
        S_.prune_rare(1.0)
    assert e.value.code == capi.DFB_ERR_INVALID and "score_only" in str(e.value)
    assert S_.table_stats() == st


# ---------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------
def test_cli_prune_rare_across_a_checkpoint(exe, tmp_path):   # noqa: F811
    data, val = str(tmp_path / "train.libsvm"), str(tmp_path / "val.libsvm")
    write_libsvm(data, 1500, 3)
    write_libsvm(val, 300, 4)
    common = [f"data_in={data}", f"data_val={val}", "V_dim=16", "l1=0", "lr=0.2", "V_threshold=0", "batch_size=50",
              "shuffle=2", "num_jobs_per_epoch=3", "stop_rel_objv=0", "stop_val_auc=-2", "table_capacity=65536",
              "num_gpus=1", "prune_period=5", "prune_count=1"]
    rare = common + ["prune_rare=1"]
    C_ = run(exe, rare + ["max_num_epochs=3", f"model_out={tmp_path / 'c.model'}"])
    assert C_.returncode == 0, C_.stderr[-2000:]
    lines = prune_lines(C_.stdout)
    freed = [int(ln.split("V rows freed ")[1].split(",")[0]) for ln in lines]
    assert len(lines) >= 5 and sum(freed) > 0, lines
    P = str(tmp_path / "ckpt")
    A = run(exe, rare + ["max_num_epochs=2", f"checkpoint_out={P}", "checkpoint_period=35"])
    assert A.returncode == 0, A.stderr[-2000:]
    assert prune_lines(A.stdout) == lines[:len(prune_lines(A.stdout))]
    B = run(exe, rare + ["max_num_epochs=3", f"checkpoint_in={P}", f"model_out={tmp_path / 'b.model'}"])
    assert B.returncode == 0, B.stderr[-2000:]
    head = B.stdout.split("Resuming from checkpoint")[1].split("\n")[0]
    epoch, m = int(head.split("epoch ")[1].split(",")[0]), int(head.split("minibatch ")[1])
    assert m % 5 == 0 and any(ln.startswith(f"Prune: minibatch {m},") for ln in lines)
    assert epoch_lines(B.stdout, epoch) == epoch_lines(C_.stdout, epoch)
    after = [ln for ln in lines if int(ln.split("minibatch ")[1].split(",")[0]) > m]
    assert after and prune_lines(B.stdout) == after, "the prunes after the checkpoint"
    assert open(tmp_path / "b.model", "rb").read() == open(tmp_path / "c.model", "rb").read()
    # refused under prune_rare = 0, given or not, by name
    for other in (common, common + ["prune_rare=0"]):
        bad = run(exe, other + [f"checkpoint_in={P}", "max_num_epochs=3"])
        assert bad.returncode != 0 and "prune_rare" in bad.stderr, bad.stderr[-2000:]
    # a checkpoint written without prune_rare (as every one before the key existed) resumes under the default only
    Q = str(tmp_path / "old")
    O = run(exe, common + ["max_num_epochs=1", f"checkpoint_out={Q}", "checkpoint_period=20"])
    assert O.returncode == 0, O.stderr[-2000:]
    assert "V rows freed" not in O.stdout
    ok = run(exe, common + ["max_num_epochs=2", f"checkpoint_in={Q}"])
    assert ok.returncode == 0 and "Resuming from checkpoint" in ok.stdout, ok.stderr[-2000:]
    bad = run(exe, rare + ["max_num_epochs=2", f"checkpoint_in={Q}"])
    assert bad.returncode != 0 and "prune_rare" in bad.stderr, bad.stderr[-2000:]
