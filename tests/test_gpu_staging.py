"""Steps on host batches and dfb_prefetch_raw: a step reuses the copy a prefetch staged only when it is given the very
batch that was prefetched -- the same nrows and the same offset, ids, value and label arrays -- and otherwise stages
its own arguments.  Every case runs an engine E and a twin T built with the same kwargs; T makes the same calls
without any prefetch, each step on fresh copies of the arrays E's step is given, so no pointer can match by accident.
After each step E and T must agree: predictions, nrows / new_keys / new_vrows / AUC of the Progress, rng_state,
table_stats and the model bit for bit; loss and penalty within 1e-6 relative (double atomicAdd sums, whose order may
vary between runs, as in test_gpu_predict.assert_same_step).  V_dim above 128 runs the generic kernels, whose float
sums are not in a fixed order (two identical runs differ in the last bits of their predictions and model): there
predictions, loss, penalty, AUC and the model's weights are held to GENERIC_TOL, far below what a step on another
batch changes.

  1. the pointer matrix on one GPU: train_step_raw (want_pred), train_step_raw_async and predict_raw_async, each
     after a prefetch that differs from the step in one argument, at V_dim 0, 16, 64 (specialised kernels) and 257
     (generic), binary and valued batches with rows at and above long_row_nnz;
  2. calls between the prefetch and the step: a device step, a host-localized step, read_progress, sync, a call
     refused by check_csr, a batch dropped for an id outside id_bits, and a second prefetch;
  3. a long pipeline: 24 async steps in flight (three times the 8-slot Progress ring) mixing training with and without
     the count push, validation and predict, binary and valued batches, pinned and pageable arrays, batches growing
     4x so that every staged buffer is reallocated under earlier steps; also on an engine that grows its table;
  4. the sharded store (ranks on one GPU, tests/shard_sim.py): the matrix of 1 through dfb_shard_step_async,
     dfb_shard_begin_async + dfb_shard_phase (one and two ranks), dfb_shard_begin_predict_async and
     dfb_shard_predict_async.

id_bits > 0 throughout: with a learned range (id_bits = 0) async and sync steps may legitimately drop different
batches (test_gpu_id_range.py).  Before a case that prefetches a batch without values and steps on it with values,
every single-GPU engine has staged valued batches at least as large into both input sets, so that an engine that
wrongly reused the prefetch would read an earlier batch's values rather than unallocated memory."""
import os
import sys
import zlib

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import oracle as O  # noqa: E402
from shard_sim import make_local  # noqa: E402
from util import assert_close, localized  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)
ID_BITS = 40
LONG = 200                     # long_row_nnz: rows of LONG or more nonzeros take the long-row kernels
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=2, V_l2=0.01, V_init_scale=0.2, seed=3,
          long_row_nnz=LONG, id_bits=ID_BITS)
B = 300
GENERIC_TOL = dict(rtol=1e-4, atol=1e-5)


def tol_of(V_dim):
    """None (bit for bit) for the specialised kernels, GENERIC_TOL above V_dim 128"""
    return None if V_dim <= 128 else GENERIC_TOL


def batch(rng, nrows, valued, id_hi=3000, row_nnz=(0, 41)):
    """nrows rows of row_nnz nonzeros, four of LONG..1.5 LONG, the last one empty (so that nrows - 1 rows hold the
    same nonzeros); ids below 2^ID_BITS"""
    nnzr = rng.integers(row_nnz[0], row_nnz[1], nrows)
    nnzr[rng.choice(nrows - 1, 4, replace=False)] = rng.integers(LONG, LONG * 3 // 2, 4)
    nnzr[-1] = 0
    off = np.concatenate([[0], np.cumsum(nnzr)]).astype(U64)
    n = int(off[-1])
    ids = (rng.integers(0, id_hi, n).astype(U64) * GOLDEN) % U64(1 << ID_BITS)
    val = (rng.random(n).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(nrows) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, ids, val, lab


def warm_batch(rng):
    """valued, more nonzeros than any batch of batch(rng, B, ...): rows of 60..80 alone hold >= 17940"""
    return batch(rng, B, True, row_nnz=(60, 81))


def copies(b):
    return tuple(None if a is None else a.copy() for a in b)


def keys_of(*batches):
    return np.unique(np.concatenate([O.localize(b[0], b[1])[1] for b in batches]))


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def pinned(n):
    return torch.zeros(max(n, 1), dtype=torch.float32, pin_memory=True)


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
def close(a, b, rtol=1e-6):
    return a == b or abs(a - b) <= rtol * max(abs(a), abs(b))


def same_progress(pe, pt, what, tol=None):
    assert (pe.nrows, pe.new_keys, pe.new_vrows) == (pt.nrows, pt.new_keys, pt.new_vrows), \
        (what, pe.as_dict(), pt.as_dict())
    rtol = 1e-6 if tol is None else tol["rtol"]
    assert (pe.auc == pt.auc if tol is None else close(pe.auc, pt.auc, rtol)), (what, pe.as_dict(), pt.as_dict())
    assert close(pe.loss, pt.loss, rtol) and close(pe.penalty, pt.penalty, rtol), (what, pe.as_dict(), pt.as_dict())


def same_pred(pe, pt, what, tol=None):
    pe, pt = np.asarray(pe), np.asarray(pt)
    assert pe.shape == pt.shape, what
    if tol is not None:
        assert_close(pe, pt, what=f"{what}: predictions", **tol)
        return
    assert np.array_equal(pe, pt), (what, int((pe != pt).sum()), float(np.abs(pe - pt).max()))


def same_model(a, b, what, tol):
    """read_entries of the same keys: bit for bit, or (tol) keys, has-V flags and feature counts exact and the
    weights, AdaGrad state and V rows within tol"""
    if tol is None:
        for x, y in zip(a, b):
            assert np.array_equal(x, y), what
        return
    (sa, ha, Va, ca), (sb, hb, Vb, cb) = a, b
    assert np.array_equal(ha, hb) and np.array_equal(sa[:, 0], sb[:, 0]), what
    for x, y, name in ((sa[:, 1:], sb[:, 1:], "w/sqrt_g/z"), (Va, Vb, "V"), (ca, cb, "cg")):
        assert_close(x, y, what=f"{what}: {name}", **tol)


def same_engine(E, T, what, capacity=True, tol=None, keys=None):
    """the InitV stream, the table counts (and capacities unless one engine grows) and the model: the snapshot bytes,
    or with tol the entries of keys (every key the engines saw)"""
    assert E.rng_state() == T.rng_state(), what
    se, st = E.table_stats(), T.table_stats()
    if not capacity:
        se, st = (se["n_keys"], se["n_vrows"]), (st["n_keys"], st["n_vrows"])
    assert se == st, (what, se, st)
    if tol is None:
        assert E.snapshot() == T.snapshot(), what
    else:
        same_model(E.read_entries(keys), T.read_entries(keys), what, tol)


def same_entries(E, T, keys, what):
    assert E.rng_state() == T.rng_state(), what
    assert E.table_stats() == T.table_stats(), what
    same_model(E.read_entries(keys), T.read_entries(keys), what, None)


def outcome(fn):
    """fn()'s result, or the DfbError code it raised: the twins must fail alike"""
    try:
        return "ok", fn()
    except capi.DfbError as e:
        return "error", e.code


# ---------------------------------------------------------------------------------------------------------------------
# one step through each entry point: (Progress, predictions or None)
# ---------------------------------------------------------------------------------------------------------------------
def step_sync(E, nrows, b, push=True, train=True):
    off, ids, val, lab = b
    assert nrows == len(off) - 1
    return E.train_step_raw(off, ids, val, lab, push_cnt=push, is_train=train, want_pred=True)


def step_async(E, nrows, b, push=True, train=True):
    off, ids, val, lab = b
    E.train_step_raw_async(nrows, off, ids, val, lab, push, train)
    return E.wait_step(), None


def step_predict(E, nrows, b, push=None, train=None):
    off, ids, val, lab = b
    out = pinned(nrows)
    E.predict_raw_async(nrows, off, ids, val, lab, out)
    pr = E.wait_step()
    return pr, out.numpy()[:nrows].copy()


ENTRIES = {"sync": step_sync, "async": step_async, "predict": step_predict}


def twins(V_dim):
    """E and T of the same model, each warmed by two valued steps (one per input set) larger than any later batch;
    returns E, T and the warm-up batches"""
    E, T = (capi.Engine(V_dim=V_dim, table_capacity=1 << 14, **KW) for _ in range(2))
    rng = np.random.default_rng(1000 + V_dim)
    warm = [warm_batch(rng) for _ in range(2)]
    for j, w in enumerate(warm):
        pe, pt = (X.train_step_raw(*copies(w), push_cnt=True, is_train=True) for X in (E, T))
        same_progress(pe, pt, f"warm-up {j}", tol_of(V_dim))
    return E, T, warm


# ---------------------------------------------------------------------------------------------------------------------
# 1. the pointer matrix
# ---------------------------------------------------------------------------------------------------------------------
def mismatch(case, rng, b):
    """(prefetch nrows, prefetch arrays, step arrays) of a case: the prefetch differs from the step in one way.
    The step is on b (or b without values / labels); the step has nrows = len(b[3])"""
    off, ids, val, lab = b
    n = len(lab)
    if case == "same":
        return n, b, b
    if case == "moved":                 # the same contents at other addresses
        return n, copies(b), b
    if case == "offset":                # the rows re-split: the same nrows and nnz, other boundaries
        nnzr = rng.permutation(np.diff(off.astype(np.int64)))
        off2 = np.concatenate([[0], np.cumsum(nnzr)]).astype(U64)
        assert off2[-1] == off[-1] and not np.array_equal(off2, off)
        return n, (off2, ids, val, lab), b
    if case == "values":
        return n, (off, ids, rng.random(len(ids)).astype(np.float32) + 1, lab), b
    if case == "values NULL->V":
        return n, (off, ids, None, lab), b
    if case == "values V->NULL":
        return n, b, (off, ids, None, lab)
    if case == "labels":
        return n, (off, ids, val, -lab), b
    if case == "labels NULL->L":
        return n, (off, ids, val, None), b
    if case == "labels L->NULL":
        return n, b, (off, ids, val, None)
    if case == "ids":                   # other ids, the same nnz
        return n, (off, (ids + U64(1) * GOLDEN) % U64(1 << ID_BITS), val, lab), b
    if case == "nrows":                 # nrows - 1: the same pointers and nnz (the last row is empty)
        assert off[-1] == off[-2]
        return n - 1, b, b
    raise ValueError(case)


CASES = ["same", "moved", "offset", "labels", "ids", "nrows"]
VALUE_CASES = ["values", "values NULL->V", "values V->NULL"]
LABEL_CASES = ["labels NULL->L", "labels L->NULL"]


def matrix(entries, V_dims):
    out = []
    for entry in entries:
        for V_dim in V_dims:
            for valued in (False, True):
                cases = CASES + (VALUE_CASES if valued else []) + (LABEL_CASES if "predict" in entry else [])
                kind = "valued" if valued else "binary"
                out += [pytest.param(entry, V_dim, valued, c, id=f"{entry}-{V_dim}-{kind}-{c}") for c in cases]
    return out


@pytest.mark.parametrize("entry,V_dim,valued,case", matrix(ENTRIES, (0, 16, 64, 257)))
def test_step_after_a_prefetch(entry, V_dim, valued, case):
    E, T, warm = twins(V_dim)
    tol = tol_of(V_dim)
    rng = np.random.default_rng(seed_of(entry, V_dim, valued, case))
    b = batch(rng, B, valued)
    n_pre, pre, st = mismatch(case, rng, b)
    keys = keys_of(*warm, b, pre)
    E.prefetch_raw(n_pre, *pre)
    # then a second step on the same arrays (the other input set): no prefetch left behind
    for what in (case, f"{case}, again"):
        pe, qe = ENTRIES[entry](E, B, st)
        pt, qt = ENTRIES[entry](T, B, copies(st))
        same_progress(pe, pt, what, tol)
        if qe is not None:
            same_pred(qe, qt, what, tol)
            assert np.any(qt != 0)
        same_engine(E, T, what, tol=tol, keys=keys)


# ---------------------------------------------------------------------------------------------------------------------
# 2. calls between the prefetch and the step
# ---------------------------------------------------------------------------------------------------------------------
def on_device(b):
    dev = torch.device("cuda", 0)
    out = tuple(None if a is None else torch.from_numpy(a.view(np.int64) if a.dtype == U64 else a).to(dev) for a in b)
    torch.cuda.synchronize()
    return out


def between(kind, X, c):
    """the call `kind` on engine X, with batch c where it takes one; returns what can be compared"""
    off, ids, val, lab = c
    n = len(lab)
    if kind == "device step":
        d = on_device(c)
        X.train_step_raw_dev(n, len(ids), d[0], d[1], d[2], d[3], False, True)
        return X.read_progress().as_dict()
    if kind == "host-localized step":
        loc = localized((off, lab, ids, val))
        X.train_step_async(n, loc["offset"], loc["lidx"], loc["value"], loc["label"], loc["keys"], len(loc["keys"]),
                           None, True)
        return X.wait_step().as_dict()
    if kind == "read_progress":
        return X.read_progress().as_dict()
    if kind == "sync":
        return X.sync()
    if kind == "refused":               # a row running backwards: check_csr refuses it before anything is staged
        bad = off.copy()
        bad[n // 2] = bad[n // 2 + 1] + U64(1)
        r = outcome(lambda: X.train_step_raw_async(n, bad, ids, val, lab, False, True))
        assert r == ("error", capi.DFB_ERR_INVALID), r
        return r
    if kind == "dropped":               # an id at 2^ID_BITS: the step is staged and submitted, then dropped
        bad = ids.copy()
        bad[len(bad) // 3] = U64(1 << ID_BITS)
        X.train_step_raw_async(n, off, bad, val, lab, False, True)
        r = outcome(X.wait_step)
        assert r == ("error", capi.DFB_ERR_INVALID), r
        return r
    raise ValueError(kind)


BETWEEN = ["device step", "host-localized step", "read_progress", "sync", "refused", "dropped"]


@pytest.mark.parametrize("entry", list(ENTRIES))
@pytest.mark.parametrize("kind", BETWEEN)
def test_call_between_prefetch_and_step(kind, entry):
    """prefetch(b); X; step(b) -- then prefetch(b); X; step(d); step(b), which puts b's step on the input set X may
    have written (an X that submits a step advances the input sets)"""
    E, T, _ = twins(16)
    rng = np.random.default_rng(seed_of(kind, entry))
    b, c, d = batch(rng, B, True), batch(rng, B, False), batch(rng, B, True)
    for seq in (("b",), ("d", "b")):
        E.prefetch_raw(B, *b)
        xe, xt = between(kind, E, c), between(kind, T, copies(c))
        assert xe == xt, (kind, xe, xt)
        for name in seq:
            st = dict(b=b, d=d)[name]
            pe, qe = ENTRIES[entry](E, B, st)
            pt, qt = ENTRIES[entry](T, B, copies(st))
            what = f"{kind}, then {seq}: step {name}"
            same_progress(pe, pt, what)
            if qe is not None:
                same_pred(qe, qt, what)
            same_engine(E, T, what)


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_second_prefetch_wins(entry):
    """prefetch(b); prefetch(c); step(c) reuses c's copy, and prefetch(b); prefetch(c); step(b) restages b"""
    E, T, _ = twins(16)
    rng = np.random.default_rng(seed_of("second prefetch", entry))
    b = batch(rng, B, True)
    c = tuple(mismatch(case, rng, b)[1][j] for j, case in enumerate(("offset", "ids", "values", "labels")))
    # (c: the same nrows and nnz as b, every array another)
    for st in (c, b):
        E.prefetch_raw(B, *b)
        E.prefetch_raw(B, *c)
        pe, qe = ENTRIES[entry](E, B, st)
        pt, qt = ENTRIES[entry](T, B, copies(st))
        what = "step on the second prefetch" if st is c else "step on the first prefetch"
        same_progress(pe, pt, what)
        if qe is not None:
            same_pred(qe, qt, what)
        same_engine(E, T, what)


# ---------------------------------------------------------------------------------------------------------------------
# 3. a long pipeline
# ---------------------------------------------------------------------------------------------------------------------
def pipeline_plan(rng, n=24):
    """(kind, push, batch, pinned, prefetch) per step: kinds cycle train+push / train / val / predict, values on every
    other step, torch pinned arrays on every third, a prefetch before every other step; nrows 150 -> 600, ids from a
    range that grows with the run so that every step brings new keys"""
    kinds = [("train", True), ("train", False), ("val", False), ("predict", False)]
    plan = []
    for j in range(n):
        kind, push = kinds[j % 4]
        nrows = 150 + 450 * j // (n - 1)
        b = batch(rng, nrows, j % 2 == 1, id_hi=3000 + 1500 * j)
        if j % 3 == 0:
            b = tuple(None if a is None else torch.from_numpy(a.view(np.int64) if a.dtype == U64 else a).pin_memory()
                      for a in b)
        plan.append((kind, push, b, j % 3 == 0, j % 2 == 0))
    return plan


def as_numpy(b):
    """fresh numpy copies of a batch held in numpy or torch arrays"""
    def one(a):
        if isinstance(a, torch.Tensor):
            a = a.numpy().view(U64) if a.dtype == torch.int64 else a.numpy()
        return a.copy()
    return tuple(None if a is None else one(a) for a in b)


@pytest.mark.parametrize("grow", [False, True], ids=["fixed", "growing"])
@pytest.mark.parametrize("V_dim", [16, 64])
def test_pipeline_past_the_progress_ring(V_dim, grow):
    if grow:
        E = capi.Engine(V_dim=V_dim, table_capacity=1 << 10, table_capacity_max=1 << 18, V_capacity_max=1 << 18, **KW)
    else:
        E = capi.Engine(V_dim=V_dim, table_capacity=1 << 17, **KW)
    T = capi.Engine(V_dim=V_dim, table_capacity=1 << 17, **KW)
    plan = pipeline_plan(np.random.default_rng(V_dim + grow))
    outs = []
    for kind, push, b, _, pre in plan:
        nrows = len(b[3])
        if pre:
            E.prefetch_raw(nrows, *b)
        if kind == "predict":
            outs.append(pinned(nrows))
            E.predict_raw_async(nrows, *b, outs[-1])
        else:
            E.train_step_raw_async(nrows, *b, push, kind == "train")
    got = [E.wait_step() for _ in range(8)]
    with pytest.raises(capi.DfbError):
        E.wait_step()
    backlog = E.read_progress()
    want, preds = [], []
    for kind, push, b, _, _ in plan:
        nb = as_numpy(b)
        if kind == "predict":
            pr, q = T.predict_raw(*nb)
            preds.append(q)
        else:
            pr = T.train_step_raw(*nb, push_cnt=push, is_train=kind == "train")
        want.append(pr)
    for j in range(8):
        same_progress(got[j], want[16 + j], f"step {16 + j}")
    old = want[:16]
    assert backlog.nrows == sum(p.nrows for p in old)
    assert backlog.new_keys == sum(p.new_keys for p in old) and backlog.new_vrows == sum(p.new_vrows for p in old)
    for f in ("loss", "penalty", "auc"):
        w = sum(float(getattr(p, f)) for p in old)
        assert abs(getattr(backlog, f) - w) <= 1e-6 * abs(w), (f, getattr(backlog, f), w)
    assert len(outs) == len(preds) == 6
    for j, (o, q) in enumerate(zip(outs, preds)):
        same_pred(o.numpy()[:len(q)], q, f"predict step {4 * j + 3}")
    same_engine(E, T, "after the pipeline", capacity=not grow)
    if grow:
        assert E.table_stats()["capacity"] < T.table_stats()["capacity"]
        assert E.growth_stats()[0] > 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. the sharded store
# ---------------------------------------------------------------------------------------------------------------------
def shard_twins(S, V_dim):
    """two stores of S ranks on one GPU, trained alike by two valued steps"""
    kw = dict(KW, V_dim=V_dim)
    E, T = (make_local(S, kw, max_rows=512, max_nnz=1 << 15) for _ in range(2))
    rng = np.random.default_rng(2000 + 10 * S + V_dim)
    for j in range(2):
        ws = [warm_batch(rng) for _ in range(S)]
        for X in (E, T):
            shard_enqueue(X, [copies(w) for w in ws], [len(w[0]) - 1 for w in ws], True, True, "begin")
            for r in range(S):
                X[r].wait_step()
    return E, T


def shard_enqueue(X, bs, nrows, push, train, entry, outs=None):
    """one step of every rank of store X: bs[r] = (off, ids, val, lab)"""
    for r, (E, b, n) in enumerate(zip(X, bs, nrows)):
        if entry == "step":
            E.shard_step_async(n, *b, push_cnt=push, is_train=train)
        elif entry == "begin":
            E.shard_begin_async(n, *b, push_cnt=push, is_train=train)
        elif entry == "begin_predict":
            E.shard_begin_predict_async(n, *b, outs[r])
        elif entry == "predict":
            E.shard_predict_async(n, *b, outs[r])
    if entry in ("begin", "begin_predict"):
        for ph in range(5):
            for E in X:
                E.shard_phase(ph)


def shard_step(X, bs, entry):
    S = len(X)
    nrows = [len(b[0]) - 1 for b in bs]
    outs = [pinned(n) for n in nrows] if "predict" in entry else None
    shard_enqueue(X, bs, nrows, True, True, entry, outs)
    prs = [X[r].wait_step() for r in range(S)]
    return prs, [None if outs is None else o.numpy()[:n].copy() for o, n in zip(outs or [None] * S, nrows)]


SHARD_ENTRIES = [("step", 1), ("begin", 1), ("begin", 2), ("begin_predict", 1), ("begin_predict", 2), ("predict", 1)]


def shard_matrix():
    out = []
    for entry, S in SHARD_ENTRIES:
        for V_dim in (0, 16, 64):
            for valued in (False, True):
                cases = CASES + (VALUE_CASES if valued else []) + (LABEL_CASES if "predict" in entry else [])
                out += [pytest.param(entry, S, V_dim, valued, c,
                                     id=f"{entry}-S{S}-{V_dim}-{'valued' if valued else 'binary'}-{c}") for c in cases]
    return out


@pytest.mark.parametrize("entry,S,V_dim,valued,case", shard_matrix())
def test_shard_step_after_a_prefetch(entry, S, V_dim, valued, case):
    """rank 0 prefetches a batch that differs from its step in one way; any other rank steps without a prefetch"""
    E, T = shard_twins(S, V_dim)
    rng = np.random.default_rng(seed_of(entry, S, V_dim, valued, case))
    bs = [batch(rng, B, valued) for _ in range(S)]
    n_pre, pre, st = mismatch(case, rng, bs[0])
    E[0].prefetch_raw(n_pre, *pre)
    steps = [st] + bs[1:]
    keys = keys_of(*bs, *([pre] if case == "ids" else []))
    for again in ("", ", again"):
        pe, qe = shard_step(E, steps, entry)
        pt, qt = shard_step(T, [copies(s) for s in steps], entry)
        for r in range(S):
            what = f"{case}{again}, rank {r}"
            same_progress(pe[r], pt[r], what)
            if qe[r] is not None:
                same_pred(qe[r], qt[r], what)
            same_entries(E[r], T[r], keys, what)
    for X in (E, T):
        for R in X:
            R.close()
