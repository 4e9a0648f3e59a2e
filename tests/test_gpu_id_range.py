"""The GPU localizer's id range (engine kwarg id_bits, or the range learned from the first raw batch), as the benchmark
and the sharded store configure it.

- Legal ranges: ids below 2^id_bits, and up to the nibble above it (the sorted range is rounded up to whole nibbles),
  sorted with 32-bit keys (id_bits <= 32) or 64-bit keys: the raw-id steps are bit-identical to the host-localized step.
- Dropped batches: a batch with an id outside the sorted range changes nothing (table, V rows, AdaGrad state, rand_r
  state), adds nothing to Progress and is reported once as DFB_ERR_INVALID, through every raw entry point and on both
  the device-count (sorted scatter) and the host-count (atomic scatter, V_dim 5) paths.
- dfb_localize measures the range of every input, whatever id_bits says, and leaves no error behind.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from util import localized

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=1, V_l2=0.02, V_init_scale=0.2, seed=5)
PROGRESS = ("loss", "penalty", "auc", "nrows", "new_keys", "new_vrows")


def nibble_top(id_bits):
    """the sorted range of an id_bits engine: ids below 2^(4 ceil(id_bits / 4))"""
    return 4 * ((id_bits + 3) // 4)


def rand_u64(rng, n, bits):
    """n uniform ids below 2^bits (bits <= 64)"""
    x = (rng.integers(0, 1 << 32, n, dtype=U64) << U64(32)) | rng.integers(0, 1 << 32, n, dtype=U64)
    return x if bits == 64 else x & U64((1 << bits) - 1)


def csr(rng, lens, ids, valued):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(U64)
    assert int(off[-1]) == len(ids)
    val = (rng.random(len(ids)).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(len(lens)) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, lab, ids, val


def on_device(batch):
    """the batch's arrays as device tensors, resident before the engine's streams read them"""
    dev = torch.device("cuda", 0)
    out = tuple(None if a is None else torch.from_numpy(a.view(np.int64) if a.dtype == U64 else a).to(dev)
                for a in batch)
    torch.cuda.synchronize()
    return out


def progress_rc(E, fn):
    """rc and Progress of dfb_read_progress / dfb_wait_step (the Python wrapper drops the Progress on an error)"""
    pr = capi.Progress()
    rc = getattr(E.L, fn)(E.h, C.byref(pr))
    return rc, pr


def as_tuple(pr):
    return tuple(getattr(pr, f) for f in PROGRESS)


def seen_keys(batches):
    """the table keys of raw batches: ReverseBytes(id % (2^64 - 1)); UINT64_MAX is not a key (it marks empty slots)"""
    ids = np.concatenate([b[2] for b in batches])
    return np.unique(O.reverse_bytes_np(np.where(ids == U64(0xFFFFFFFFFFFFFFFF), U64(0), ids)))


def assert_same_model(A, B, keys):
    for x, y in zip(A.read_entries(keys), B.read_entries(keys)):
        assert np.array_equal(x, y)
    assert A.table_stats() == B.table_stats()
    assert A.rng_state() == B.rng_state()


# ---------------------------------------------------------------------------------------------------------------------
# legal ranges
# ---------------------------------------------------------------------------------------------------------------------
def range_batch(rng, id_bits, B=3000, valued=False):
    """rows of 1..40 ids (over 20 emit tiles of 2048 pairs) drawn from a pool of at most ~600 ids (key runs of ~100 pairs
    that cross tile boundaries): 0, 2^id_bits - 1, ids below 2^id_bits and ids in [2^id_bits, 2^nibble_top) -- the
    rounding of the range to whole nibbles accepts those"""
    top = nibble_top(id_bits)
    pool = [np.array([0, (1 << id_bits) - 1], U64), rand_u64(rng, 400, id_bits)]
    if top > id_bits:
        span = (1 << top) - (1 << id_bits)
        pool.append(U64(1 << id_bits) + rand_u64(rng, 200, 64) % U64(span))
        pool.append(np.array([(1 << top) - 1, 1 << id_bits], U64))
    pool = np.unique(np.concatenate(pool))
    lens = rng.integers(1, 41, B)
    ids = pool[rng.integers(0, len(pool), int(lens.sum()))]
    ids[np.cumsum(lens)[:-1]] = 0                     # 0 (the id) in every row but the first: one run across all tiles
    return csr(rng, lens, ids, valued)


@pytest.mark.parametrize("id_bits", [1, 4, 13, 16, 29, 30, 31, 32, 33, 36, 40, 48, 63, 64])
def test_id_bits_range_raw_steps_equal_localized_step(id_bits):
    rng = np.random.default_rng(100 + id_bits)
    kw = dict(V_dim=16, table_capacity=1 << 14, **KW)
    batches = [range_batch(rng, id_bits, valued=j == 1) for j in range(2)]
    assert all(int(b[0][-1]) > 20 * 2048 for b in batches)
    D = capi.Engine(id_bits=id_bits, **kw)        # device-resident batches: no synchronisation inside the step
    S = capi.Engine(id_bits=id_bits, **kw)        # synchronous dfb_train_step_raw: also sorts within id_bits
    L = capi.Engine(**kw)                         # host-localized
    devb = [on_device(b) for b in batches]
    for ep in range(2):
        for (o, l, i, v), (do, dl, di, dv) in zip(batches, devb):
            b = localized((o, l, i, v))
            pl = L.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"] if ep == 0 else None, True)
            D.train_step_raw_dev(len(l), len(i), do, di, dv, dl, ep == 0, True)
            pd = D.read_progress()
            ps = S.train_step_raw(o, i, v, l, push_cnt=(ep == 0), is_train=True)
            assert as_tuple(pd) == as_tuple(pl) and as_tuple(ps) == as_tuple(pl)
    keys = seen_keys(batches)
    assert_same_model(D, L, keys)
    assert_same_model(S, L, keys)
    for (o, l, i, v) in batches:
        gl, gk, gc = D.localize(o, i)
        ol, ok, oc = O.localize(o, i)
        assert np.array_equal(gl, ol) and np.array_equal(gk, ok) and np.array_equal(gc, oc)


# ---------------------------------------------------------------------------------------------------------------------
# dropped batches
# ---------------------------------------------------------------------------------------------------------------------
def drop_batches(rng, id_bits, valued):
    """legal batches over a shared pool of ids below 2^id_bits, every id at most once per batch (so that the atomic
    scatter adds one term per key and is bit-reproducible too); 'bad' batches are legal ones plus one id 2^nibble_top,
    the smallest id outside the sorted range, appended to their last row.  The second bad batch is larger than any
    batch before it (the workspaces grow for it)."""
    pool = np.unique(rand_u64(rng, 6000, id_bits))

    def one(rows, bad, j):
        lens = rng.integers(1, 16, rows)
        ids = rng.choice(pool, int(lens.sum()), replace=False)
        if bad:
            ids = np.concatenate([ids, np.array([1 << nibble_top(id_bits)], U64)])
            lens[-1] += 1
        return csr(rng, lens, ids, valued and j % 2 == 1)

    seq = [("bad", one(60, True, 0))]
    seq += [("ok", one(80, False, j)) for j in range(1, 4)]
    seq += [("bad", one(400, True, 4))]
    seq += [("ok", one(80, False, j)) for j in range(5, 7)]
    assert int(seq[4][1][0][-1]) > max(int(b[0][-1]) for _, b in seq[:4])
    return seq


@pytest.mark.parametrize("entry", ["sync", "async", "dev"])
@pytest.mark.parametrize("scatter,V_dim", [("sorted", 64), ("atomic", 5)])   # device- / host-side key count
@pytest.mark.parametrize("id_bits", [16, 30, 32, 36])
def test_batch_outside_id_bits_is_dropped(id_bits, scatter, V_dim, entry):
    rng = np.random.default_rng(7 * id_bits + V_dim)
    seq = drop_batches(rng, id_bits, valued=True)
    kw = dict(V_dim=V_dim, scatter=scatter, id_bits=id_bits, table_capacity=1 << 14, **KW)
    E = capi.Engine(**kw)
    T = capi.Engine(**kw)          # the twin never sees the bad batches
    keys = seen_keys([b for _, b in seq])       # incl. the rejected id's key
    zero = (0.0,) * 4 + (0, 0)
    pending = []                   # async: (kind, twin Progress) per submitted step

    def run(X, o, l, i, v, push):
        """one step; returns (rc, Progress) for the sync / dev entry points, None for async (collected later)"""
        if entry == "sync":
            pr = capi.Progress()
            rc = X.L.dfb_train_step_raw(X.h, len(l), capi._p(o), capi._p(i), capi._p(v), capi._p(l), int(push), 1,
                                        C.byref(pr), None)
            return rc, pr
        if entry == "async":
            X.train_step_raw_async(len(l), o, i, v, l, push_cnt=push)
            return None
        do, dl, di, dv = on_device((o, l, i, v))
        X.train_step_raw_dev(len(l), len(i), do, di, dv, dl, push, True)
        return progress_rc(X, "dfb_read_progress")       # synchronises: the inputs may be freed afterwards

    for t, (kind, (o, l, i, v)) in enumerate(seq):
        push = t < 3
        got = run(E, o, l, i, v, push)
        if entry == "async":
            rc, pr = progress_rc(E, "dfb_wait_step")
        else:
            rc, pr = got
        if kind == "bad":
            assert rc == capi.DFB_ERR_INVALID, f"step {t}: rc {rc}"
            msg = E.L.dfb_last_error(E.h).decode()
            assert "id_bits = %d" % id_bits in msg and "2^%d" % nibble_top(id_bits) in msg, msg
            assert as_tuple(pr) == zero                                  # adds nothing to any Progress field
            if entry != "sync":
                assert as_tuple(E.read_progress()) == zero               # the next read is clean
        else:
            assert rc == 0, f"step {t}: {E.L.dfb_last_error(E.h).decode()}"
            tw = run(T, o, l, i, v, push)
            if entry == "async":
                tw = progress_rc(T, "dfb_wait_step")
            assert tw[0] == 0
            assert as_tuple(pr) == as_tuple(tw[1]), f"step {t}"
        assert_same_model(E, T, keys)
    E.sync()
    assert as_tuple(E.read_progress()) == zero


# ---------------------------------------------------------------------------------------------------------------------
# the learned range (no id_bits)
# ---------------------------------------------------------------------------------------------------------------------
def learned_batch(rng, lo_bits, hi_bits, rows=120, valued=False, const=None):
    lens = rng.integers(1, 30, rows)
    n = int(lens.sum())
    if const is not None:
        ids = np.full(n, const, U64)
    else:
        ids = rand_u64(rng, n, hi_bits)
        if lo_bits:                                         # half of the ids at or above 2^lo_bits
            ids[::2] |= U64(1 << lo_bits)
    return csr(rng, lens, ids, valued)


@pytest.mark.parametrize("entry", ["async", "dev"])
@pytest.mark.parametrize("case", ["12_to_40", "32_to_33", "all_zero", "all_max"])
def test_learned_range_drops_wider_batch_then_widens(case, entry):
    """the first batch fixes the range; a wider one is dropped and reported, and its mask (read back after the
    step) widens the range, so that after a sync the same kind of batch is accepted; narrower batches always are"""
    rng = np.random.default_rng(len(case) * 31 + len(entry))
    if case == "12_to_40":
        first, wide, narrow = learned_batch(rng, 0, 12), learned_batch(rng, 39, 40), learned_batch(rng, 0, 12)
    elif case == "32_to_33":       # 32-bit sort keys (k_rev_keys<true> keeps only the upper half); the OR mask sees all
        first, wide, narrow = learned_batch(rng, 0, 32), learned_batch(rng, 32, 33), learned_batch(rng, 0, 30)
    else:                          # lowest_bit of an all-zero mask is 63: every id but 0 / UINT64_MAX is outside
        c = 0 if case == "all_zero" else 0xFFFFFFFFFFFFFFFF
        first, wide, narrow = learned_batch(rng, 0, 0, const=c), learned_batch(rng, 0, 20), learned_batch(rng, 0, 0, const=c)
    kw = dict(V_dim=16, table_capacity=1 << 14, **KW)
    E = capi.Engine(**kw)
    L = capi.Engine(**kw)          # host-localized twin: never sees the dropped batch
    wide2 = learned_batch(rng, 39 if case == "12_to_40" else 32 if case == "32_to_33" else 0,
                          40 if case == "12_to_40" else 33 if case == "32_to_33" else 20, valued=True)
    seq = [("ok", first), ("bad", wide), ("sync", None), ("ok", wide2), ("ok", narrow), ("ok", wide)]
    keys = seen_keys([b for _, b in seq if b is not None])
    t = 0
    for kind, batch in seq:
        if kind == "sync":
            E.sync()
            continue
        o, l, i, v = batch
        if entry == "async":
            E.train_step_raw_async(len(l), o, i, v, l, push_cnt=True)
            rc, pr = progress_rc(E, "dfb_wait_step")
        else:
            do, dl, di, dv = on_device(batch)
            E.train_step_raw_dev(len(l), len(i), do, di, dv, dl, True, True)
            rc, pr = progress_rc(E, "dfb_read_progress")
        if kind == "bad":
            assert rc == capi.DFB_ERR_INVALID
            assert "id_bits = 0" in E.L.dfb_last_error(E.h).decode()
            assert as_tuple(pr) == (0.0,) * 4 + (0, 0)
        else:
            assert rc == 0, f"step {t}: {E.L.dfb_last_error(E.h).decode()}"
            b = localized(batch)
            pl = L.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"], True)
            assert as_tuple(pr) == as_tuple(pl), f"step {t}"
        assert_same_model(E, L, keys)
        t += 1


# ---------------------------------------------------------------------------------------------------------------------
# dfb_localize on an id_bits engine
# ---------------------------------------------------------------------------------------------------------------------
def test_localize_ignores_id_bits_and_leaves_no_error():
    rng = np.random.default_rng(3)
    kw = dict(V_dim=16, id_bits=16, table_capacity=1 << 14, **KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)
    o, l, i, v = learned_batch(rng, 0, 16, rows=3000)
    i[::5] = rand_u64(rng, len(i[::5]), 40)                  # ids far above 2^16 (and over 20 emit tiles)
    gl, gk, gc = E.localize(o, i)
    ol, ok, oc = O.localize(o, i)
    assert np.array_equal(gl, ol) and np.array_equal(gk, ok) and np.array_equal(gc, oc)
    legal = learned_batch(rng, 0, 16)
    pe = E.train_step_raw(legal[0], legal[2], legal[3], legal[1], push_cnt=True)     # reads back clean
    pt = T.train_step_raw(legal[0], legal[2], legal[3], legal[1], push_cnt=True)
    assert as_tuple(pe) == as_tuple(pt)
    assert_same_model(E, T, seen_keys([legal]))
