"""The streamed checkpoint (dfb_snapshot_write / dfb_restore_read): the v1 byte format against an independent numpy
encoder, round trips, re-sharding M parts into N ranks, the cleared-table error contract, and the CLI's model_in of
a sharded model on one GPU.  The shard tests run S ranks on one GPU (tests/shard_sim.py)."""
import io
import os
import struct
import subprocess
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import oracle as O  # noqa: E402
from shard_sim import all_keys, check_progress, key_owner_np, make_local, raw_batch, run_local  # noqa: E402
from util import localized, rand_batch  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(V_dim=16, l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)
MAGIC = b"DFB200\x00\x01"


# ---------------------------------------------------------------------------------------------------------------------
# an independent encoder / walker of format v1
# ---------------------------------------------------------------------------------------------------------------------
def encode_v1(E, keys, save_aux):
    """the expected snapshot of engine E, whose keys are all in `keys`, from read_entries / rng_state / table_stats"""
    keys = np.unique(np.asarray(keys, np.uint64))
    scal, hasv, V, cg = E.read_entries(keys)
    st = E.table_stats()
    present = hasv >= 0
    assert present.sum() == st["n_keys"], "the key list must cover the table"
    out = bytearray(struct.pack("<8sIiQQII", MAGIC, 1, E.V_dim, st["n_keys"], st["n_vrows"], E.rng_state(),
                                1 if save_aux else 0))
    for i in np.nonzero(present)[0]:
        out += struct.pack("<Q", int(keys[i]))
        out += scal[i, :2].astype("<f4").tobytes()
        if save_aux:
            out += scal[i, 2:].astype("<f4").tobytes()
        out += struct.pack("<i", int(hasv[i]))
        if hasv[i] == 1:
            out += V[i].astype("<f4").tobytes()
            if save_aux:
                out += cg[i].astype("<f4").tobytes()
    return bytes(out)


def record_offsets(blob, V_dim):
    """byte offset and has_V of every record"""
    aux = struct.unpack_from("<I", blob, 36)[0] == 1
    fixed = 28 if aux else 20
    row = V_dim * 4 * (2 if aux else 1)
    pos, out = 40, []
    while pos < len(blob):
        hv = struct.unpack_from("<i", blob, pos + fixed - 4)[0]
        out.append((pos, hv))
        pos += fixed + (row if hv else 0)
    assert pos == len(blob)
    return out, fixed


class Sink:
    def __init__(self, limit):
        self.parts, self.limit = [], limit

    def write(self, b):
        assert len(b) <= self.limit, (len(b), self.limit)
        self.parts.append(bytes(b))

    def value(self):
        return b"".join(self.parts)


class SmallReads(io.BytesIO):
    """a source that hands out odd-sized pieces (records straddle every boundary)"""
    def read(self, n=-1):
        return super().read(min(n, 333) if n and n > 0 else n)


def streamed(E, save_aux=True, chunk=0):
    s = Sink(chunk or 64 << 20)
    E.snapshot_to(s, save_aux=save_aux, chunk_bytes=chunk)
    return s.value()


def train(E, batches, first_cnt=True):
    for j, b in enumerate(batches):
        E.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"],
                     b["cnt"] if (first_cnt and j < 2) else None, True)


# ---------------------------------------------------------------------------------------------------------------------
# 1. format oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim,with_v", [(0, False), (10, True), (64, True), (64, False), (128, True)])
def test_snapshot_bytes_equal_the_numpy_encoder(V_dim, with_v):
    rng = np.random.default_rng(40 + V_dim)
    kw = dict(KW, V_dim=V_dim, V_threshold=1 if with_v else 10 ** 6)
    batches = [localized(rand_batch(rng, 150, 20, 900, j % 2 == 0)) for j in range(4)]
    E = capi.Engine(table_capacity=1 << 14, **kw)
    train(E, batches)
    st = E.table_stats()
    assert st["n_keys"] > 300 and ((st["n_vrows"] > 100) == with_v)
    keys = np.unique(np.concatenate([b["keys"] for b in batches]))
    for aux in (False, True):
        want = encode_v1(E, keys, aux)
        assert E.snapshot(save_aux=aux) == want
        for chunk in (1000, 4096, 0):
            assert streamed(E, aux, chunk) == want, (aux, chunk)


def test_snapshot_of_one_bin_larger_than_a_pass():
    """ids that are multiples of 2^24 (so also of 2^20): every reversed key has its top 24 bits zero and falls into
    the same top-20-bit bin, far larger than the pass budget a 1000-byte chunk gives"""
    rng = np.random.default_rng(5)
    kw = dict(KW, V_dim=16, V_threshold=0)
    ids_space = 3000
    batches = [localized(rand_batch(rng, 200, 20, ids_space, True, mult=1 << 24)) for _ in range(3)]
    keys = np.unique(np.concatenate([b["keys"] for b in batches]))
    assert len(np.unique(keys >> np.uint64(44))) == 1
    E = capi.Engine(table_capacity=1 << 14, **kw)
    train(E, batches)
    assert E.table_stats()["n_keys"] > 1000
    want = encode_v1(E, keys, True)
    assert streamed(E, True, 1000) == want
    F = capi.Engine(table_capacity=1 << 14, **kw)
    F.restore_from(io.BytesIO(want), chunk_bytes=1000)
    for x, y in zip(E.read_entries(keys), F.read_entries(keys)):
        assert np.array_equal(x, y)


# ---------------------------------------------------------------------------------------------------------------------
# 2. round trip
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [0, 16])
def test_restore_from_stream_round_trip_and_resume(V_dim):
    rng = np.random.default_rng(31 + V_dim)
    kw = dict(KW, V_dim=V_dim, seed=6)
    batches = [localized(rand_batch(rng, 200, 25, 600, j % 2 == 0)) for j in range(6)]
    keys = np.unique(np.concatenate([b["keys"] for b in batches]))
    A = capi.Engine(table_capacity=1 << 14, **kw)
    train(A, batches[:3])
    buf = io.BytesIO()
    A.snapshot_to(buf, chunk_bytes=1000)
    assert buf.getvalue() == A.snapshot()
    B = capi.Engine(table_capacity=1 << 14, **kw)
    assert B.restore_from(SmallReads(buf.getvalue()), chunk_bytes=1000) is True
    assert B.table_stats() == A.table_stats() and B.rng_state() == A.rng_state()
    for x, y in zip(A.read_entries(keys), B.read_entries(keys)):
        assert np.array_equal(x, y)
    for b in batches[3:]:
        pa = A.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, True)
        pb = B.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, True)
        assert pa.loss == pb.loss and pa.penalty == pb.penalty
    for x, y in zip(A.read_entries(keys), B.read_entries(keys)):
        assert np.array_equal(x, y)
    assert A.rng_state() == B.rng_state() and streamed(A, True, 4096) == streamed(B, True, 4096)
    # without aux data: predicts like A, refuses to train
    C2 = capi.Engine(table_capacity=1 << 14, **kw)
    noaux = io.BytesIO()
    A.snapshot_to(noaux, save_aux=False, chunk_bytes=1000)
    assert C2.restore_from(io.BytesIO(noaux.getvalue()), chunk_bytes=1000) is False
    b = batches[0]
    assert (C2.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, False).loss
            == A.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, False).loss)
    with pytest.raises(capi.DfbError):
        C2.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, True)
    with pytest.raises(capi.DfbError):
        C2.snapshot_to(io.BytesIO(), save_aux=True)


# ---------------------------------------------------------------------------------------------------------------------
# 3. re-sharding
# ---------------------------------------------------------------------------------------------------------------------
STEPS = 5


def batch_fn(rank, step):
    return raw_batch(rank, step, valued=(step % 2 == 0), ids=700)


def parts_of(engines, chunk=1000):
    out = []
    for E in engines:
        buf = io.BytesIO()
        E.snapshot_to(buf, chunk_bytes=chunk)
        out.append(buf.getvalue())
    return out


def overlaps(p, M, r, N):
    def rng_(i, S):
        w = (2 ** 64 - 1) // S
        return w * i, (2 ** 64 - 1 if i == S - 1 else w * (i + 1) - 1)
    plo, phi = rng_(p, M)
    rlo, rhi = rng_(r, N)
    return plo <= rhi and rlo <= phi


def restore_parts(engines, parts):
    N, M = len(engines), len(parts)
    for r, E in enumerate(engines):
        for p in range(M):
            if overlaps(p, M, r, N):
                E.restore_from(io.BytesIO(parts[p]), part=p, nparts=M, shard=r, nshards=N, chunk_bytes=1000)


@pytest.mark.parametrize("S", [2, 3])
def test_parts_merge_into_one_engine_and_reshard(S):
    engines, _ = run_local(S, KW, STEPS, batch_fn)
    keys = all_keys(S, STEPS, batch_fn)
    own = key_owner_np(keys, S)
    ref = [E.read_entries(keys) for E in engines]
    stats = [E.table_stats() for E in engines]
    parts = parts_of(engines)
    # all parts -> one engine
    one = capi.Engine(table_capacity=1 << 15, **KW)
    restore_parts([one], parts)
    got = one.read_entries(keys)
    for s in range(S):
        m = own == s
        for x, y in zip(got, ref[s]):
            assert np.array_equal(x[m], y[m])
    st = one.table_stats()
    assert st["n_keys"] == sum(x["n_keys"] for x in stats) and st["n_vrows"] == sum(x["n_vrows"] for x in stats)
    assert one.rng_state() == engines[0].rng_state()        # the lowest part read
    # S parts -> N ranks (2 -> 3, 3 -> 2)
    N = 3 if S == 2 else 2
    re = make_local(N, KW)
    restore_parts(re, parts)
    nown = key_owner_np(keys, N)
    for r in range(N):
        x = re[r].read_entries(keys)
        assert np.all(x[1][nown != r] == -1)
        for a, b in zip(x, got):
            assert np.array_equal(a[nown == r], b[nown == r])
        assert re[r].table_stats()["n_keys"] == (nown == r).sum()
    # a validation step of the re-sharded store == the one-engine restore's prediction, per worker
    vfn = lambda r, step: batch_fn(r, 100 + step)          # noqa: E731
    _, prog = run_local(N, KW, 1, vfn, train_fn=lambda step: False, cnt_steps=0, engines=re)
    for r in range(N):
        off, idx, val, lab = vfn(r, 0)
        pr = one.train_step_raw(off, idx, val, lab, push_cnt=False, is_train=False)
        check_progress(prog[r][0], [pr.loss, pr.penalty, pr.auc, 0, pr.nrows], f"re-shard {S}->{N} worker {r}")


def test_same_count_restore_resumes_the_sharded_run_bitwise():
    S = 2
    full, _ = run_local(S, KW, STEPS + 3, batch_fn)
    half, _ = run_local(S, KW, STEPS, batch_fn)
    parts = parts_of(half)
    resumed = make_local(S, KW)
    restore_parts(resumed, parts)
    for r in range(S):
        assert resumed[r].rng_state() == half[r].rng_state()
    run_local(S, KW, 3, lambda r, st: batch_fn(r, STEPS + st), cnt_steps=0, engines=resumed)
    keys = all_keys(S, STEPS + 3, batch_fn)
    for r in range(S):
        for x, y in zip(full[r].read_entries(keys), resumed[r].read_entries(keys)):
            assert np.array_equal(x, y)
        assert full[r].rng_state() == resumed[r].rng_state()
        assert full[r].table_stats() == resumed[r].table_stats()


# ---------------------------------------------------------------------------------------------------------------------
# 4. errors: the table is cleared and the engine restores and trains afterwards
# ---------------------------------------------------------------------------------------------------------------------
class FailingReader(io.BytesIO):
    def read(self, n=-1):
        if self.tell() > 0:
            raise OSError("disk gone")
        return super().read(n)


class FailingWriter:
    def __init__(self):
        self.n = 0

    def write(self, b):
        self.n += 1
        if self.n > 2:
            raise OSError("disk full")


def test_restore_errors_clear_the_table():
    rng = np.random.default_rng(77)
    batches = [localized(rand_batch(rng, 200, 20, 800, j % 2 == 0)) for j in range(3)]
    A = capi.Engine(table_capacity=1 << 14, **KW)
    train(A, batches)
    blob = A.snapshot()
    recs, fixed = record_offsets(blob, KW["V_dim"])
    assert len(recs) > 200
    mid = len(recs) // 2
    jv = next(j for j in range(mid, len(recs)) if recs[j][1] == 1)

    def patched(off, word):
        b = bytearray(blob)
        b[off:off + len(word)] = word
        return bytes(b)

    key_j = blob[recs[mid][0]:recs[mid][0] + 8]
    cases = {
        "truncated header": blob[:20],
        "truncated mid-record": blob[:recs[mid][0] + 6],
        "truncated mid-row": blob[:recs[jv][0] + fixed + 8],
        "has_V flipped": patched(recs[mid][0] + fixed - 4, struct.pack("<i", 2)),
        "has_V 1 -> 0": patched(recs[jv][0] + fixed - 4, struct.pack("<i", 0)),
        "keys not ascending": patched(recs[mid + 1][0], key_j),
    }
    E = capi.Engine(table_capacity=1 << 14, **KW)
    b = batches[0]

    def cleared(what, code=capi.DFB_ERR_INVALID):
        assert E.table_stats()["n_keys"] == 0, what
        return True

    for what, data in cases.items():
        with pytest.raises(capi.DfbError) as ei:
            E.restore_from(io.BytesIO(data), chunk_bytes=1000)
        assert ei.value.code == capi.DFB_ERR_INVALID and "cleared" in str(ei.value), (what, str(ei.value))
        cleared(what)
    # wrong V_dim
    with pytest.raises(capi.DfbError):
        capi.Engine(table_capacity=1 << 14, **dict(KW, V_dim=8)).restore_from(io.BytesIO(blob))
    # the same part twice
    E.restore_from(io.BytesIO(blob), chunk_bytes=1000)
    assert E.table_stats()["n_keys"] == A.table_stats()["n_keys"]
    with pytest.raises(capi.DfbError) as ei:
        E.restore_from(io.BytesIO(blob), chunk_bytes=1000)
    assert "cleared" in str(ei.value)
    cleared("twice")
    # a key outside the declared part: part 0 of 2 read as part 1 of 2
    own = key_owner_np(np.unique(np.concatenate([x["keys"] for x in batches])), 2)
    assert (own == 0).any()
    with pytest.raises(capi.DfbError) as ei:
        E.restore_from(io.BytesIO(blob), part=1, nparts=2, chunk_bytes=1000)
    assert "outside part" in str(ei.value)
    cleared("part range")
    # table_capacity too small
    small = capi.Engine(table_capacity=100, **KW)
    with pytest.raises(capi.DfbError) as ei:
        small.restore_from(io.BytesIO(blob), chunk_bytes=1000)
    assert ei.value.code == capi.DFB_ERR_CAPACITY
    assert small.table_stats()["n_keys"] == 0
    # source error
    with pytest.raises(capi.DfbError):
        E.restore_from(FailingReader(blob), chunk_bytes=1000)
    cleared("source")
    # the engine restores and trains afterwards
    assert E.restore_from(io.BytesIO(blob), chunk_bytes=1000) is True
    pa = A.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, True)
    pe = E.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, True)
    assert pa.loss == pe.loss
    # a sink error fails the snapshot and changes nothing: the model is still there, a second snapshot works
    before = A.table_stats()
    with pytest.raises(capi.DfbError):
        A.snapshot_to(FailingWriter(), chunk_bytes=1000)
    assert A.table_stats() == before
    assert streamed(A, True, 1000) == A.snapshot()
    with pytest.raises(capi.DfbError):               # dfb_restore keeps refusing a non-empty table, clearing nothing
        A.restore(blob)
    assert A.table_stats() == before


# ---------------------------------------------------------------------------------------------------------------------
# 5. CLI: a model written in 2 parts, predicted on one GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_bin():
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    return hb.build()


def write_libsvm(path, rows, seed):
    rng = np.random.default_rng(seed)
    with open(path, "w") as f:
        for _ in range(rows):
            ids = np.unique(rng.integers(1, 3000, rng.integers(3, 30)))
            x = (rng.random(len(ids)) + 0.25).astype(np.float32)
            f.write(f"{1 if rng.random() < 0.4 else -1} " + " ".join(f"{int(i)}:{v:.9g}" for i, v in zip(ids, x)) + "\n")


def read_libsvm(path):
    off, idx, val, lab = [0], [], [], []
    for line in open(path):
        t = line.split()
        lab.append(float(t[0]))
        for kv in t[1:]:
            i, v = kv.split(":")
            idx.append(int(i))
            val.append(np.float32(v))
        off.append(len(idx))
    return (np.array(off, np.uint64), np.array(idx, np.uint64), np.array(val, np.float32),
            np.array(lab, np.float32))


def cli_kw():
    return ["V_dim=16", "l1=0.05", "l2=0.01", "lr=0.2", "V_lr=0.1", "V_threshold=1", "V_l2=0.01", "V_init_scale=0.2",
            "seed=3", "batch_size=100", "table_capacity=16384"]


def test_cli_predicts_a_two_part_model_on_one_gpu(host_bin, tmp_path):
    data = str(tmp_path / "d.libsvm")
    write_libsvm(data, 600, 9)
    off, idx, val, lab = read_libsvm(data)

    def fn(rank, step):        # rank r, step t: rows [100 (2 t + r), +100)
        r0 = 100 * (2 * step + rank)
        o = off[r0:r0 + 101]
        return (o - o[0], idx[int(o[0]):int(o[-1])], val[int(o[0]):int(o[-1])], lab[r0:r0 + 100])

    engines, _ = run_local(2, KW, 3, fn)
    base = str(tmp_path / "model")
    for r, blob in enumerate(parts_of(engines)):
        with open(f"{base}_part-{r}", "wb") as f:
            f.write(blob)
    preds = str(tmp_path / "pred.txt")
    out = subprocess.run([os.path.join(host_bin, "difacto_b200"), "task=predict", "num_gpus=1", f"model_in={base}",
                          f"data_in={data}", f"pred_out={preds}"] + cli_kw(), capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "Loaded model" in out.stdout and "2 parts" in out.stdout
    got = np.loadtxt(preds, dtype=np.float32)
    one = capi.Engine(table_capacity=1 << 14, **KW)
    restore_parts([one], parts_of(engines))
    _, want = one.train_step_raw(off, idx, val, lab, push_cnt=False, is_train=False, want_pred=True)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_cli_train_and_predict_on_different_gpu_counts(host_bin, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    exe = os.path.join(host_bin, "difacto_b200")
    data = str(tmp_path / "d.libsvm")
    write_libsvm(data, 2000, 4)

    def loss(out):
        assert out.returncode == 0, out.stderr[-2000:]
        return float(out.stdout.split("Prediction: loss = ")[1].split(",")[0])

    def run(args):
        return subprocess.run([exe, f"data_in={data}"] + cli_kw() + args, capture_output=True, text=True, timeout=300)

    for train_gpus, pred_gpus in ((2, 1), (1, 2)):
        model = str(tmp_path / f"m{train_gpus}")
        out = run(["max_num_epochs=2", f"num_gpus={train_gpus}", f"model_out={model}"])
        assert out.returncode == 0, out.stderr[-2000:]
        same = loss(run(["task=predict", f"num_gpus={train_gpus}", f"model_in={model}"]))
        other_args = ["task=predict", f"num_gpus={pred_gpus}", f"model_in={model}"]
        if pred_gpus == 1:
            other_args.append(f"pred_out={tmp_path / 'p.txt'}")
        other = loss(run(other_args))
        assert other == pytest.approx(same, rel=1e-4)
