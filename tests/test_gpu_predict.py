"""Predict steps on raw ids (dfb_predict_raw_async / _dev, dfb_shard_*predict*, task=predict): the forward pass of a
frozen model.  On one GPU its predictions must be bit-identical to the validation step's (train_step_raw with
is_train=False) while writing nothing of the model; the sharded store's must match one engine holding the merged
model.  The shard tests run S ranks on one GPU (tests/shard_sim.py)."""
import io
import os
import subprocess
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from shard_sim import make_local, raw_batch, run_local  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=2, V_l2=0.01, V_init_scale=0.2, seed=3)


def mixed_batch(rng, B, valued, id_lo=0, id_hi=600, long_nnz=200, id_bits=64):
    """rows of 0..40 nonzeros, a few of long_nnz..1.5 long_nnz (the long-row kernel's), ids id_lo..id_hi spread over
    the whole reversed key space (below 2^id_bits)"""
    nnzr = rng.integers(0, 41, B)
    nnzr[rng.choice(B, 4, replace=False)] = rng.integers(long_nnz, long_nnz * 3 // 2, 4)
    off = np.concatenate([[0], np.cumsum(nnzr)]).astype(np.uint64)
    n = int(off[-1])
    ids = rng.integers(id_lo, id_hi, n).astype(np.uint64) * GOLDEN
    if id_bits < 64:
        ids %= np.uint64(1 << id_bits)
    val = (rng.random(n).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, ids, val, lab


def trained(V_dim, rng, steps=4, **kw):
    """ids 0..5999, about 2 occurrences each per batch: with V_threshold 2 some keys get a V row, some do not"""
    E = capi.Engine(V_dim=V_dim, table_capacity=1 << 14, long_row_nnz=200, **dict(KW, **kw))
    for s in range(steps):
        off, ids, val, lab = mixed_batch(rng, 300, s % 2 == 0, id_hi=6000, id_bits=kw.get("id_bits") or 64)
        E.train_step_raw(off, ids, val, lab, push_cnt=s < 2, is_train=True)
    return E


def assert_same_step(pp, vp, what):
    """a predict step's Progress against the validation step's: AUC equal, loss within 1e-6, no penalty"""
    assert pp.auc == vp.auc, (what, pp.auc, vp.auc)
    assert pp.loss == vp.loss or abs(pp.loss - vp.loss) <= 1e-6 * abs(vp.loss), (what, pp.loss, vp.loss)
    assert pp.nrows == vp.nrows and pp.penalty == 0 and pp.new_keys == 0 and pp.new_vrows == 0, what


def pinned(n):
    return torch.zeros(max(n, 1), dtype=torch.float32, pin_memory=True)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bit identity with the validation step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [0, 3, 8, 10, 16, 40, 64, 128])
@pytest.mark.parametrize("valued", [False, True])
def test_predictions_are_bitwise_the_validation_step(V_dim, valued):
    rng = np.random.default_rng(V_dim * 2 + valued)
    E = trained(V_dim, rng)
    st = E.table_stats()
    assert st["n_keys"] > 400 and (V_dim == 0 or 0 < st["n_vrows"] < st["n_keys"])     # keys with and without V
    off, ids, val, lab = mixed_batch(rng, 400, valued, id_hi=8000)                       # ids >= 6000: not in the table
    pp, pred = E.predict_raw(off, ids, val, lab)
    vp, want = E.train_step_raw(off, ids, val, lab, push_cnt=False, is_train=False, want_pred=True)
    assert np.array_equal(pred, want), (V_dim, valued, np.abs(pred - want).max())
    assert_same_step(pp, vp, (V_dim, valued))
    assert np.any(pred != 0)


# ---------------------------------------------------------------------------------------------------------------------
# 2. read-only
# ---------------------------------------------------------------------------------------------------------------------
def test_predict_writes_nothing_of_the_model():
    rng = np.random.default_rng(5)
    E = trained(16, rng)
    F = trained(16, np.random.default_rng(5))
    before = (E.snapshot(), E.table_stats(), E.rng_state())
    for j in range(3):      # full of ids the table has never seen
        off, ids, val, lab = mixed_batch(rng, 200, j % 2 == 0, id_lo=10 ** 6, id_hi=10 ** 6 + 5000)
        pr, pred = E.predict_raw(off, ids, val, lab)
        assert np.all(pred == 0) and pr.nrows == 200 and pr.new_keys == 0
    assert (E.snapshot(), E.table_stats(), E.rng_state()) == before
    # a training step afterwards: the same model as on the engine that never predicted
    off, ids, val, lab = mixed_batch(rng, 300, True, id_hi=800)
    pe = E.train_step_raw(off, ids, val, lab, is_train=True)
    pf = F.train_step_raw(off, ids, val, lab, is_train=True)
    assert pe.loss == pf.loss and pe.new_keys == pf.new_keys
    assert E.snapshot() == F.snapshot() and E.rng_state() == F.rng_state()


# ---------------------------------------------------------------------------------------------------------------------
# 3. pipelining
# ---------------------------------------------------------------------------------------------------------------------
def test_ten_outstanding_predict_steps():
    rng = np.random.default_rng(11)
    E = trained(64, rng)
    batches = [mixed_batch(rng, 150 + 10 * j, j % 2 == 1, id_hi=700) for j in range(10)]
    want = [E.predict_raw(*b) for b in batches]
    outs = [pinned(len(b[3])) for b in batches]
    for b, o in zip(batches, outs):
        E.predict_raw_async(len(b[3]), b[0], b[1], b[2], b[3], o)
    # the Progress ring holds 8 steps: the two oldest are folded into what read_progress returns
    got = [E.wait_step() for _ in range(8)]
    with pytest.raises(capi.DfbError):
        E.wait_step()
    backlog = E.read_progress()
    assert backlog.nrows == want[0][0].nrows + want[1][0].nrows
    for j in range(10):
        assert np.array_equal(outs[j].numpy()[:len(batches[j][3])], want[j][1]), j
    for j in range(8):
        assert got[j].nrows == want[j + 2][0].nrows and got[j].auc == want[j + 2][0].auc, j


def test_predict_steps_see_the_training_steps_before_them():
    rng = np.random.default_rng(12)
    E, F = trained(32, rng), trained(32, np.random.default_rng(12))
    tr = [mixed_batch(rng, 300, j % 2 == 0) for j in range(3)]
    pv = [mixed_batch(rng, 200, j % 2 == 1, id_hi=700) for j in range(3)]
    outs = [pinned(200) for _ in range(3)]
    for t, p, o in zip(tr, pv, outs):
        E.train_step_raw_async(len(t[3]), t[0], t[1], t[2], t[3], False, True)
        E.predict_raw_async(len(p[3]), p[0], p[1], p[2], p[3], o)
    for t, p, o in zip(tr, pv, outs):
        E.wait_step()
        pp = E.wait_step()
        F.train_step_raw(*t, is_train=True)
        vp, want = F.train_step_raw(*p, is_train=False, want_pred=True)
        assert np.array_equal(o.numpy(), want)
        assert_same_step(pp, vp, "interleaved")


def test_prefetched_predict_step_and_null_labels():
    rng = np.random.default_rng(13)
    E = trained(8, rng)
    off, ids, val, lab = mixed_batch(rng, 250, True, id_hi=700)
    _, want = E.train_step_raw(off, ids, val, lab, is_train=False, want_pred=True)
    out = pinned(250)
    E.prefetch_raw(250, off, ids, val, None)
    E.predict_raw_async(250, off, ids, val, None, out)
    pr = E.wait_step()
    assert np.array_equal(out.numpy(), want)
    assert pr.loss == 0 and pr.auc == 0 and pr.nrows == 250 and pr.penalty == 0
    pr2, pred = E.predict_raw(off, ids, val, None)
    assert np.array_equal(pred, want) and pr2.loss == 0 and pr2.nrows == 250


def test_predict_raw_dev_matches_the_host_form():
    rng = np.random.default_rng(14)
    E = trained(10, rng)
    off, ids, val, lab = mixed_batch(rng, 300, False, id_hi=700)
    _, want = E.predict_raw(off, ids, val, lab)
    d = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()   # noqa: E731
    d_pred = torch.zeros(300, device="cuda")
    E.predict_raw_dev(300, len(ids), d(off), d(ids), None, d(lab), d_pred)
    pr = E.read_progress()
    assert np.array_equal(d_pred.cpu().numpy(), want) and pr.nrows == 300 and pr.penalty == 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. edge cases
# ---------------------------------------------------------------------------------------------------------------------
def test_id_bits_drop():
    rng = np.random.default_rng(15)
    E = trained(16, rng, id_bits=40)
    off, ids, val, lab = mixed_batch(rng, 200, True, id_hi=700, id_bits=40)
    good = (off, ids, val, lab)
    bad_ids = ids.copy()
    bad_ids[7] = np.uint64(1 << 41)
    out = pinned(200)
    out.fill_(1.0)
    E.predict_raw_async(200, off, bad_ids, val, lab, out)
    with pytest.raises(capi.DfbError) as ei:
        E.wait_step()
    assert ei.value.code == capi.DFB_ERR_INVALID and "id_bits = 40" in str(ei.value)
    assert np.all(out.numpy() == 0)
    pr = E.read_progress()                   # once: the drop added nothing, and is not reported again
    assert pr.nrows == 0 and pr.loss == 0 and pr.auc == 0
    pp, pred = E.predict_raw(*good)
    vp, want = E.train_step_raw(*good, is_train=False, want_pred=True)
    assert np.array_equal(pred, want) and pp.nrows == 200


@pytest.mark.parametrize("kw", [dict(V_dim=129), dict(V_dim=16, force_generic=1)])
def test_fallback_widths_equal_the_validation_step(kw):
    rng = np.random.default_rng(16)
    E = capi.Engine(table_capacity=1 << 14, long_row_nnz=200, **dict(KW, **kw))
    for s in range(3):
        E.train_step_raw(*mixed_batch(rng, 200, s % 2 == 0), push_cnt=s < 2, is_train=True)
    snap = E.snapshot()
    off, ids, val, lab = mixed_batch(rng, 200, True, id_hi=800)
    pp, pred = E.predict_raw(off, ids, val, lab)
    vp, want = E.train_step_raw(off, ids, val, lab, is_train=False, want_pred=True)
    assert np.array_equal(pred, want)
    assert_same_step(pp, vp, kw)
    assert E.snapshot() == snap


def test_a_sharded_engine_refuses_predict_raw():
    engines = make_local(2, dict(KW, V_dim=8))
    off, ids, val, lab = raw_batch(0, 0, True)
    with pytest.raises(capi.DfbError) as ei:
        engines[0].predict_raw(off, ids, val, lab)
    assert ei.value.code == capi.DFB_ERR_INVALID
    d = torch.zeros(1, device="cuda")
    with pytest.raises(capi.DfbError):
        engines[1].predict_raw_dev(0, 0, d, d, None, None, None)


# ---------------------------------------------------------------------------------------------------------------------
# 5. predictions out of the sharded store
# ---------------------------------------------------------------------------------------------------------------------
def overlaps(p, M, r, N):
    def rng_(i, S):
        w = (2 ** 64 - 1) // S
        return w * i, (2 ** 64 - 1 if i == S - 1 else w * (i + 1) - 1)
    plo, phi = rng_(p, M)
    rlo, rhi = rng_(r, N)
    return plo <= rhi and rlo <= phi


def merged(engines, kw):
    """one engine holding every rank's part of the model"""
    one = capi.Engine(table_capacity=1 << 15, **kw)
    M = len(engines)
    for p, E in enumerate(engines):
        buf = io.BytesIO()
        E.snapshot_to(buf, chunk_bytes=1000)
        if overlaps(p, M, 0, 1):
            one.restore_from(io.BytesIO(buf.getvalue()), part=p, nparts=M, chunk_bytes=1000)
    return one


@pytest.mark.parametrize("S", [1, 2, 3])
@pytest.mark.parametrize("V_dim", [0, 10, 64])
def test_sharded_predictions_match_one_engine(S, V_dim):
    kw = dict(KW, V_dim=V_dim)
    fn = lambda r, st: raw_batch(r, st, valued=(st % 2 == 0), ids=600, mixed=True, B=96)   # noqa: E731
    engines, _ = run_local(S, kw, 4, fn, max_rows=128, max_nnz=16384)
    one = merged(engines, kw)
    snaps = [E.snapshot() for E in engines]
    for step, valued in ((10, False), (11, True)):
        batches = [raw_batch(r, step, valued, ids=900, mixed=True, B=96) for r in range(S)]
        outs = [pinned(96) for _ in range(S)]
        for r, (E, (off, ids, val, lab)) in enumerate(zip(engines, batches)):
            # rank 0 of a multi-rank store predicts without labels
            E.shard_begin_predict_async(96, off, ids, val, None if (r == 0 and S > 1) else lab, outs[r])
        for ph in range(5):
            for E in engines:
                E.shard_phase(ph)
        for r, (E, (off, ids, val, lab)) in enumerate(zip(engines, batches)):
            pr = E.wait_step()
            vp, want = one.predict_raw(off, ids, val, lab)
            got = outs[r].numpy()
            assert np.all(np.abs(got - want) <= 1e-5 + 1e-5 * np.abs(want)), (S, V_dim, r, np.abs(got - want).max())
            assert pr.nrows == 96 and pr.penalty == 0 and pr.new_keys == 0
            if r == 0 and S > 1:
                assert pr.loss == 0 and pr.auc == 0
            else:       # (V_dim 0 leaves the prediction unclamped: a loss may be inf on both sides)
                assert pr.loss == vp.loss or abs(pr.loss - vp.loss) <= 1e-4 * abs(vp.loss) + 1e-4
    assert [E.snapshot() for E in engines] == snaps


def test_shard_predict_async_is_the_phased_step():
    """dfb_shard_predict_async (all five phases in one call) on a one-rank store"""
    kw = dict(KW, V_dim=16)
    fn = lambda r, st: raw_batch(r, st, valued=True, ids=500)   # noqa: E731
    engines, _ = run_local(1, kw, 3, fn)
    one = merged(engines, kw)
    off, ids, val, lab = raw_batch(0, 20, True, ids=700)
    out = pinned(len(lab))
    engines[0].shard_predict_async(len(lab), off, ids, val, lab, out)
    pr = engines[0].wait_step()
    _, want = one.predict_raw(off, ids, val, lab)
    assert np.all(np.abs(out.numpy()[:len(lab)] - want) <= 1e-5 + 1e-5 * np.abs(want)) and pr.penalty == 0


# ---------------------------------------------------------------------------------------------------------------------
# 6. CLI: task=predict pred_out=
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_bin():
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    return hb.build()


CLI_KW = dict(V_dim=16, l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=2, V_l2=0.01, V_init_scale=0.2, seed=3)


def write_rows(path, rng, rows):
    """libsvm rows of 1..9 valued features (ids < 5000); returns the CSR arrays as the reader parses them"""
    nnzr = rng.integers(1, 10, rows)
    off = np.concatenate([[0], np.cumsum(nnzr)]).astype(np.uint64)
    n = int(off[-1])
    ids = rng.integers(0, 5000, n).astype(np.uint64)
    val = (rng.integers(1, 200, n) / 64.0).astype(np.float32)        # exact in %.9g
    lab = np.where(rng.random(rows) < 0.4, 1.0, -1.0).astype(np.float32)
    with open(path, "w") as f:
        for r in range(rows):
            a, b = int(off[r]), int(off[r + 1])
            f.write(("1" if lab[r] > 0 else "-1") + "".join(f" {i}:{v:.9g}" for i, v in zip(ids[a:b], val[a:b])) + "\n")
    return off, ids, val, lab


def test_cli_predict_writes_the_validation_predictions_in_row_order(host_bin, tmp_path):
    rng = np.random.default_rng(21)
    data = str(tmp_path / "d.libsvm")
    rows = 3 * 65536 + 1234
    off, ids, val, lab = write_rows(data, rng, rows)
    E = capi.Engine(table_capacity=1 << 14, **CLI_KW)
    for s in range(3):
        a = 5000 * s
        o = off[a:a + 5001] - off[a]
        E.train_step_raw(o, ids[int(off[a]):int(off[a + 5000])], val[int(off[a]):int(off[a + 5000])], lab[a:a + 5000],
                         push_cnt=s < 2, is_train=True)
    model = str(tmp_path / "m.dfb")
    with open(model, "wb") as f:
        f.write(E.snapshot())
    preds = str(tmp_path / "p.txt")
    args = [os.path.join(host_bin, "difacto_b200"), "task=predict", f"data_in={data}", f"model_in={model}",
            f"pred_out={preds}", "batch_size=100", "table_capacity=16384"] + [f"{k}={v}" for k, v in CLI_KW.items()]
    out = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    got = np.loadtxt(preds, dtype=np.float32)
    want, want_loss = [], 0.0
    for a in range(0, rows, 65536):
        b = min(rows, a + 65536)
        o = off[a:b + 1] - off[a]
        pr, p = E.train_step_raw(o, ids[int(off[a]):int(off[b])], val[int(off[a]):int(off[b])], lab[a:b],
                                 is_train=False, want_pred=True)
        want.append(p)
        want_loss += pr.loss
    want = np.concatenate(want)
    assert got.shape == want.shape and np.array_equal(got, want)
    loss = float(out.stdout.split("Prediction: loss = ")[1].split(",")[0])
    assert abs(loss - want_loss) <= 1e-4 * want_loss


def test_cli_sharded_predict_writes_the_rows_in_file_order(host_bin, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rng = np.random.default_rng(22)
    data = str(tmp_path / "d.libsvm")
    write_rows(data, rng, 20000)
    exe = os.path.join(host_bin, "difacto_b200")
    common = [f"data_in={data}", "batch_size=500", "table_capacity=65536"] + [f"{k}={v}" for k, v in CLI_KW.items()]
    model = str(tmp_path / "m")
    out = subprocess.run([exe] + common + ["max_num_epochs=2", "num_gpus=2", f"model_out={model}"], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    p1, p2 = str(tmp_path / "p1.txt"), str(tmp_path / "p2.txt")
    for n, p in ((1, p1), (2, p2)):
        out = subprocess.run([exe] + common + ["task=predict", f"num_gpus={n}", f"model_in={model}", f"pred_out={p}"],
                             capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]
    a, b = np.loadtxt(p1, dtype=np.float32), np.loadtxt(p2, dtype=np.float32)
    assert a.shape == b.shape == (20000,)
    assert np.all(np.abs(a - b) <= 1e-5 + 1e-5 * np.abs(a))
    assert not any(f.startswith("p2.txt.part") for f in os.listdir(tmp_path))
