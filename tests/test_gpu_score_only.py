"""The scoring-only engine (score_only = 1, V_storage = fp32 | bf16): a model restored without its AdaGrad state into
V-only rows, and scored with the raw-id predict step.

Pinned here: the fp32 scoring engine gives the training engine's predict step bit for bit; the bf16 scoring engine gives,
bit for bit, what the fp32 scoring engine gives on a model whose V values were rounded to bf16 (nearest, ties to even)
beforehand, and stays within a stated bound of the CPU oracle on the unrounded model; the row pool takes 1/2 and 1/4 of
the training engine's memory; restores grow the engine and re-shard; everything that trains, reads or writes rows,
saves, prunes or shards is refused by name and changes nothing; dropped batches and the CLI behave as on the training
engine's predict path."""
import ctypes as C
import functools
import io
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

import test_gpu_id_range as idr
import test_gpu_lookup_free_step as tlf
from util import localized

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=2, V_l2=0.02, V_init_scale=0.2, seed=11,
          long_row_nnz=200, hot_split=64, id_bits=64)
CAP = dict(table_capacity=1 << 15)
GRID = [(V_dim, valued) for V_dim in (0, 5, 10, 16, 24, 64, 100, 128) for valued in (False, True)]
MAGIC = b"DFB200\x00\x01"

# V bit patterns whose bf16 rounding tells nearest-even from truncation: just below 1.0 (rounds up across a power of
# two), exact ties with an even and with an odd kept mantissa, positive and negative denormals (one an exact tie)
CRAFTED = np.array([0x3F7FFFFF, 0x3F808000, 0x3F818000, 0x00000001, 0x00018000, 0x807FFFFF, 0xBF7F8000, 0x3F7F7FFF],
                   np.uint32)


def engine(V_dim, score=None, **kw):
    """a training engine, or score = "fp32" / "bf16": a scoring-only one"""
    extra = {} if score is None else dict(score_only=True, V_storage=score)
    return capi.Engine(V_dim=V_dim, **{**CAP, **KW, **kw, **extra})


def bf16_rne(u):
    """fp32 bit patterns rounded to bf16, nearest with ties to even, as fp32 bit patterns (no NaN among them)"""
    u = u.astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32)


def v_rows(blob, V_dim):
    """a writable copy of snapshot v1 `blob` and the byte offset of every record's V[V_dim]"""
    from test_gpu_checkpoint import record_offsets
    recs, fixed = record_offsets(blob, V_dim)
    return np.frombuffer(blob, np.uint8).copy(), [pos + fixed for pos, hv in recs if hv]


def crafted(blob, V_dim):
    """the snapshot with CRAFTED written over one V value in each of its first V rows (cg untouched)"""
    a, rows = v_rows(blob, V_dim)
    for j, (at, bits) in enumerate(zip(rows, CRAFTED)):
        a[at + 4 * (j % V_dim): at + 4 * (j % V_dim) + 4] = np.frombuffer(struct.pack("<I", int(bits)), np.uint8)
    return a.tobytes()


def rounded(blob, V_dim):
    """the snapshot with every V value rounded to bf16 (cg untouched)"""
    a, rows = v_rows(blob, V_dim)
    for at in rows:
        v = a[at:at + 4 * V_dim].view(np.uint32)
        v[:] = bf16_rne(v)
    return a.tobytes()


@functools.lru_cache(maxsize=None)
def model(V_dim, valued, id_bits=64):
    """(snapshot with aux, snapshot without, scoring batches): a model trained on ids of a pool of 3000, and batches
    over a pool twice as wide (half their ids are not in the model) with rows of 0..40 and of 200..300 nonzeros"""
    rng = np.random.default_rng(100 * V_dim + valued)
    pool = np.unique(rng.integers(0, 1 << 40, 6000).astype(U64) * GOLDEN)
    if id_bits < 64:
        pool = np.unique(pool & U64((1 << id_bits) - 1))
    A = engine(V_dim, id_bits=id_bits)
    for s in range(4):
        o, l, i, v = tlf.batch(rng, pool[:3000], B=500, valued=valued, hot=pool[3])
        A.train_step_raw(o, i, v, l, s < 2, True)
    if V_dim:
        assert A.table_stats()["n_vrows"] > len(CRAFTED)
    aux, noaux = A.snapshot(True), A.snapshot(False)
    if V_dim:
        aux, noaux = crafted(aux, V_dim), crafted(noaux, V_dim)
    score = [tlf.batch(rng, pool, B=300, valued=valued, hot=pool[3]), tlf.batch(rng, pool, B=40, valued=valued)]
    return aux, noaux, score


def score(E, b):
    o, l, i, v = b
    pr, q = E.predict_raw(o, i, v, l)
    return idr.as_tuple(pr), q.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# 1. fp32 scoring = the training engine's predict step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim,valued", GRID)
def test_fp32_scoring_is_bitwise_the_training_engines_predict_step(V_dim, valued):
    aux, noaux, batches = model(V_dim, valued)
    for blob in (aux, noaux):
        T, S = engine(V_dim), engine(V_dim, "fp32")
        T.restore(blob)
        assert S.restore(blob) is False                    # has_aux of a scoring engine reads 0
        assert S.table_stats() == T.table_stats()
        for b in batches:
            want = score(T, b)
            assert want[0][3] == len(b[1]) and want[0][0] > 0
            assert score(S, b) == want


# ---------------------------------------------------------------------------------------------------------------------
# 2. bf16 scoring = fp32 scoring on the model rounded beforehand
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim,valued", GRID)
def test_bf16_scoring_is_bitwise_fp32_scoring_of_the_rounded_model(V_dim, valued):
    aux, noaux, batches = model(V_dim, valued)
    for blob in (aux, noaux):
        pre = rounded(blob, V_dim) if V_dim else blob
        if V_dim:
            assert pre != blob
            a, rows = v_rows(pre, V_dim)                    # the crafted values went where nearest-even sends them
            got = [int(a[at + 4 * (j % V_dim): at + 4 * (j % V_dim) + 4].view(np.uint32)[0])
                   for j, at in enumerate(rows[:len(CRAFTED)])]
            assert got == [0x3F800000, 0x3F800000, 0x3F820000, 0, 0x00020000, 0x80800000, 0xBF800000, 0x3F7F0000]
        F, H = engine(V_dim, "fp32"), engine(V_dim, "bf16")
        F.restore(pre)
        H.restore_from(io.BytesIO(blob), chunk_bytes=4096)
        for b in batches:
            assert score(H, b) == score(F, b)
        if V_dim >= 10 and blob is aux:                     # and rounding did change the predictions
            U = engine(V_dim, "fp32")
            U.restore(blob)
            assert score(U, batches[0])[1] != score(H, batches[0])[1]


# ---------------------------------------------------------------------------------------------------------------------
# 3. bf16 scoring against the CPU oracle on the unrounded model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim,valued", [(10, True), (64, False), (64, True), (100, True)])
def test_bf16_scoring_is_close_to_the_oracle(V_dim, valued):
    """The FM score is sum x w + sum_{i<j} x_i x_j <V_i, V_j>.  bf16 keeps 8 significant bits: a rounded V element is
    V (1 + d) with |d| <= 2^-9, so a pair's inner product moves by at most (2^-8 + 2^-18) sum_c |V_ic V_jc|, and the
    score by at most that times S = sum_{i<j} |x_i x_j| <|V_i|, |V_j|> (w is not rounded; the clamp to [-20, 20] only
    shrinks a difference).  The bound below is 2^-7 S, twice that, plus 1e-4 (1 + |score|) for the fp32 summation of
    rows of up to 300 nonzeros on either side."""
    aux, _, batches = model(V_dim, valued)
    T, H = engine(V_dim), engine(V_dim, "bf16")
    T.restore(aux)
    H.restore(aux)
    for b in batches:
        o, l, i, v = b
        loc = localized(b)
        got = np.frombuffer(score(H, b)[1], np.float32)
        scal, hasv, V, _ = T.read_entries(loc["keys"])
        vals, lens = T.pull(loc["keys"])                    # (inserts the missing keys into T: read after read_entries)
        w_pos, V_pos = O.get_pos(lens)
        want = O.fm_predict(V_dim, o, loc["lidx"], v, vals, w_pos, V_pos)
        absV = np.where((hasv == 1)[:, None], np.abs(V.astype(np.float64)), 0.0)
        x = np.ones(len(i)) if v is None else np.abs(v.astype(np.float64))
        for r in range(len(l)):
            a, e = int(o[r]), int(o[r + 1])
            rows = x[a:e, None] * absV[loc["lidx"][a:e]]
            S = 0.5 * ((rows.sum(0) ** 2).sum() - (rows ** 2).sum())
            assert abs(float(got[r]) - float(want[r])) <= 2.0 ** -7 * S + 1e-4 * (1 + abs(float(want[r]))), (r, S)


# ---------------------------------------------------------------------------------------------------------------------
# 4. memory
# ---------------------------------------------------------------------------------------------------------------------
def test_row_pool_takes_a_half_and_a_quarter():
    """300000 keys with a V row at V_dim 64 (a snapshot without aux written with numpy): 153.6 / 76.8 / 38.4 MB of rows"""
    n, k = 300000, 64
    rng = np.random.default_rng(41)
    keys = np.unique(rng.integers(0, 1 << 63, n + 1000).astype(U64))[:n]
    rec = np.zeros(n, np.dtype([("key", "<u8"), ("cnt", "<f4"), ("w", "<f4"), ("hv", "<i4"), ("V", "<f4", (k,))]))
    assert rec.dtype.itemsize == 20 + 4 * k
    rec["key"], rec["cnt"], rec["hv"] = keys, 5, 1
    rec["w"] = rng.normal(0, 0.1, n)
    rec["V"] = rng.normal(0, 0.05, (n, k))
    blob = struct.pack("<8sIiQQII", MAGIC, 1, k, n, n, 7, 0) + rec.tobytes()
    ids = O.reverse_bytes_np(keys[rng.integers(0, n, 30 * 2000)])
    b = idr.csr(rng, np.full(2000, 30), ids, True)

    def held(storage):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        E = engine(k, storage, table_capacity=1 << 19, V_capacity=n)
        E.restore(blob)
        out = score(E, b)
        E.sync()
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
        per_row, in_use = E.row_bytes()
        E.close()
        return used, per_row, in_use, out

    held(None)                                             # first use of every code path (module load, pools)
    used_t, row_t, use_t, out_t = held(None)
    used_f, row_f, use_f, out_f = held("fp32")
    used_h, row_h, use_h, out_h = held("bf16")
    assert (row_t, row_f, row_h) == (8 * k, 4 * k, 2 * k)
    assert (use_t, use_f, use_h) == (n * 8 * k, n * 4 * k, n * 2 * k)
    assert out_f == out_t and out_h[0][3] == 2000
    gran = 2 << 20                                         # each pool is mapped in whole 2 MiB pieces
    assert used_t - used_f >= (use_t - use_f) - gran, (used_t, used_f)
    assert used_f - used_h >= (use_f - use_h) - gran, (used_f, used_h)


# ---------------------------------------------------------------------------------------------------------------------
# 5. growth and re-sharding
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "bf16"])
def test_two_parts_into_three_growing_scoring_engines(storage):
    from test_gpu_checkpoint import restore_parts
    V_dim = 16
    aux, _, batches = model(V_dim, True)
    parts = []
    for r in range(2):                   # the model as two ranks of a 2-GPU run would have saved it
        P = engine(V_dim)
        P.restore_from(io.BytesIO(aux), shard=r, nshards=2)
        parts.append(P.snapshot())
    one = engine(V_dim, storage)
    one.restore(aux)
    grow = [engine(V_dim, storage, table_capacity=1024, table_capacity_max=1 << 20) for _ in range(3)]
    restore_parts(grow, parts)
    st = [g.table_stats() for g in grow]
    assert sum(s["n_keys"] for s in st) == one.table_stats()["n_keys"]
    assert sum(s["n_vrows"] for s in st) == one.table_stats()["n_vrows"]
    assert max(s["capacity"] for s in st) > 1024 and max(s["v_capacity"] for s in st) > 1024
    o, l, i, v = batches[0]
    own = O.owner(O.reverse_bytes_np(i.copy()), 3)
    rows = np.repeat(np.arange(len(l)), np.diff(o).astype(np.int64))
    for r, g in enumerate(grow):         # the batch cut down to the ids rank r owns
        keep = own == r
        b = (np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=len(l)))]).astype(U64), l, i[keep],
             v[keep])
        assert score(g, b) == score(one, b)


def test_restore_beyond_V_capacity_max_leaves_an_empty_table():
    aux, _, batches = model(16, True)
    E = engine(16, "bf16", table_capacity=1024, table_capacity_max=1 << 20, V_capacity=8, V_capacity_max=16)
    with pytest.raises(capi.DfbError) as e:
        E.restore_from(io.BytesIO(aux), chunk_bytes=4096)
    assert e.value.code == capi.DFB_ERR_CAPACITY and "cleared" in str(e.value)
    st = E.table_stats()
    assert st["n_keys"] == 0 and st["n_vrows"] == 0
    o, l, i, v = batches[1]
    assert not E.predict_raw(o, i, v, l)[1].any()           # nothing to score with: 0 for every row


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "bf16"])
def test_everything_but_restore_and_predict_is_refused_by_name(storage):
    aux, _, batches = model(16, True)
    E = engine(16, storage)
    E.restore(aux)
    b = batches[1]
    o, l, i, v = b
    loc = localized(b)
    before = score(E, b)
    st = E.table_stats()
    k1, f1, i1 = np.ones(1, U64), np.ones(17, np.float32), np.full(1, 17, np.int32)
    sink = io.BytesIO()
    calls = dict(
        train_step=lambda: E.train_step(o, loc["lidx"], v, l, loc["keys"], loc["cnt"], True),
        validation_step=lambda: E.train_step(o, loc["lidx"], v, l, loc["keys"], None, False),
        train_step_async=lambda: E.train_step_async(len(l), o, loc["lidx"], v, l, loc["keys"], len(loc["keys"])),
        train_step_dev=lambda: E.train_step_dev(0, 0, None, None, None, None, None, 0),
        train_step_raw=lambda: E.train_step_raw(o, i, v, l, True, True),
        validation_step_raw=lambda: E.train_step_raw(o, i, v, l, False, False),
        train_step_raw_async=lambda: E.train_step_raw_async(len(l), o, i, v, l),
        train_step_raw_dev=lambda: E.train_step_raw_dev(0, 0, None, None, None, None),
        push_feacnt=lambda: E.push_feacnt(k1, f1[:1]),
        pull=lambda: E.pull(k1),
        push_grad=lambda: E.push_grad(k1, f1, i1),
        predict=lambda: E.predict(o, loc["lidx"], v, f1),
        calc_grad=lambda: E.calc_grad(o, loc["lidx"], v, l, f1, np.zeros(len(l), np.float32)),
        read_entries=lambda: E.read_entries(k1),
        dev_feacnt=lambda: E.dev_feacnt(None, 0, None),
        dev_pull_rows=lambda: E.dev_pull_rows(None, 0, None, None, None),
        dev_fm_step=lambda: E.dev_fm_step(0, 0, None, None, None, None, 0, None, None, None, False, None, None),
        dev_push_rows=lambda: E.dev_push_rows(None, 0, None, None, None),
        snapshot=lambda: E.snapshot(),
        snapshot_without_aux=lambda: E.snapshot(False),
        dfb_snapshot=lambda: E._ck(E.L.dfb_snapshot(E.h, 0, (C.c_ubyte * 64)(), 64)),
        snapshot_to=lambda: E.snapshot_to(sink, save_aux=False),
        snapshot_begin=lambda: E.snapshot_begin(False),
        prune=lambda: E.prune(0.0),
        shard_init=lambda: E.shard_init(0, 1, 128, 4096),
    )
    for name, call in calls.items():
        with pytest.raises(capi.DfbError) as e:
            call()
        assert e.value.code == capi.DFB_ERR_INVALID and "score_only" in str(e.value), (name, str(e.value))
    assert sink.getvalue() == b""
    assert E.table_stats() == st and score(E, b) == before


def test_parameter_checks():
    for kw in (dict(V_dim=16, V_storage="bf16"), dict(V_dim=16, V_storage="bf16", score_only=0),
               dict(V_dim=16, score_only=1, V_storage="fp16"), dict(V_dim=129, score_only=1),
               dict(V_dim=16, score_only=1, force_generic=1), dict(V_dim=16, score_only=2)):
        with pytest.raises(capi.DfbError) as e:
            capi.Engine(**kw)
        assert e.value.code == capi.DFB_ERR_PARAM, kw
    E = capi.Engine(V_dim=16, score_only=0, V_storage="fp32")     # the defaults, spelled out: a training engine
    assert E.row_bytes()[0] == 8 * 16 and E.unknown_kwargs() == []


# ---------------------------------------------------------------------------------------------------------------------
# 7. dropped batches
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "bf16"])
def test_a_batch_outside_id_bits_is_dropped_as_on_the_training_engine(storage):
    aux, _, batches = model(16, True, id_bits=40)
    T, S = engine(16, id_bits=40), engine(16, storage, id_bits=40)
    T.restore(aux)
    S.restore(aux)
    o, l, i, v = batches[0]
    bad = i.copy()
    bad[7] = U64(1 << 41)
    for E in (T, S):
        out = torch.ones(len(l), dtype=torch.float32).pin_memory()
        E.predict_raw_async(len(l), o, bad, v, l, out)
        with pytest.raises(capi.DfbError) as e:
            E.wait_step()
        assert e.value.code == capi.DFB_ERR_INVALID and "id_bits = 40" in str(e.value)
        assert not out.numpy().any()
        assert idr.as_tuple(E.read_progress()) == (0, 0, 0, 0, 0, 0)      # reported once, and nothing added
    if storage == "fp32":
        assert score(S, batches[0]) == score(T, batches[0])
    else:
        assert score(S, batches[0])[0][3] == len(l)


# ---------------------------------------------------------------------------------------------------------------------
# 8. CLI
# ---------------------------------------------------------------------------------------------------------------------
def test_cli_predict_with_score_only(tmp_path):
    from test_gpu_checkpoint import cli_kw, read_libsvm, write_libsvm
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    exe = os.path.join(hb.build(), "difacto_b200")
    data, model_fn = str(tmp_path / "d.libsvm"), str(tmp_path / "m.dfb")
    write_libsvm(data, 1500, 13)
    off, idx, val, lab = read_libsvm(data)
    kw = dict(kv.split("=") for kv in cli_kw() if not kv.startswith(("batch_size", "table_capacity")))
    A = capi.Engine(table_capacity=1 << 14, **kw)
    for s in range(3):
        a, e = int(off[500 * s]), int(off[500 * s + 500])
        A.train_step_raw(off[500 * s:500 * s + 501] - off[500 * s], idx[a:e], val[a:e], lab[500 * s:500 * s + 500],
                         s < 2, True)
    assert A.table_stats()["n_vrows"] > 100
    with open(model_fn, "wb") as f:
        f.write(A.snapshot())

    def run(extra, name):
        out = subprocess.run([exe, "task=predict", f"model_in={model_fn}", f"data_in={data}",
                              f"pred_out={tmp_path / name}"] + cli_kw() + extra, capture_output=True, text=True,
                             timeout=300)
        return out, (open(tmp_path / name, "rb").read() if out.returncode == 0 else None)

    base, want = run([], "p0")
    assert base.returncode == 0, base.stderr[-2000:]
    so, got = run(["score_only=1"], "p1")
    assert so.returncode == 0, so.stderr[-2000:]
    assert got == want and "without aux data" in so.stdout and "unrecognized" not in so.stderr
    bf, got16 = run(["score_only=1", "V_storage=bf16"], "p2")
    assert bf.returncode == 0, bf.stderr[-2000:]
    p, q = np.loadtxt(io.BytesIO(want), dtype=np.float32), np.loadtxt(io.BytesIO(got16), dtype=np.float32)
    # the bound of test_bf16_scoring_is_close_to_the_oracle with |V| <= vmax, |x| <= 1.25 and at most 29 nonzeros a row:
    # S <= C(29, 2) 1.25^2 V_dim vmax^2
    vmax = float(np.abs(A.read_entries(np.unique(O.reverse_bytes_np(idx.copy())))[2]).max())
    assert p.shape == q.shape == (1500,) and got16 != want
    assert np.abs(p - q).max() <= 2.0 ** -7 * 406 * 1.5625 * 16 * vmax * vmax + 1e-3
    for extra in (["num_gpus=2", "score_only=1"], ["V_storage=bf16"]):
        out, _ = run(extra, "p3")
        assert out.returncode != 0 and ("score_only" in out.stderr), out.stderr[-500:]
