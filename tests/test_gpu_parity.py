"""GPU parity tests: the CUDA path (through the C-ABI) against the oracle on the same inputs.

Tolerances (fp32; the GPU uses FMA and a different summation order than the reference):
  pred          |d| <= 1e-5 + 1e-5*|ref|         (SURVEY.md 8d)
  gradients     |d| <= 2e-6 + 1e-4*|ref|         (fp32 atomics reorder the per-key sums)
  model state   |d| <= 1e-5 + 1e-3*|ref| after T steps; bit-exact when fed identical gradients
  keys / lens / w_pos / V_pos / owner shard / InitV random stream: bit-exact
"""
import numpy as np
import pytest

from conftest import parse_kwargs, syn_batches
from oracle import oracle as O
from util import assert_close, localized, oracle_state, rand_batch

pytestmark = pytest.mark.gpu

capi = pytest.importorskip("difacto_b200.capi")

PRED_TOL = dict(rtol=1e-5, atol=1e-5)
GRAD_TOL = dict(rtol=1e-4, atol=2e-6)
STATE_TOL = dict(rtol=1e-3, atol=1e-5)


def engine(**kw):
    kw.setdefault("table_capacity", 1 << 16)
    return capi.Engine(**kw)


# ----------------------------------------------------------------------------------------
# (A) Loss: FMLoss::Predict / CalcGrad on the reference's own fixture and goldens
# ----------------------------------------------------------------------------------------
def test_fm_loss_nov_golden(rcv1, refout):
    E = engine(V_dim=0)
    lidx = refout["loc_lidx"]
    w = refout["nov_w"]
    pred = E.predict(rcv1["offset"], lidx, rcv1["value"], w)
    assert_close(pred, refout["nov_pred"], what="pred", **PRED_TOL)
    assert abs(E.evaluate(rcv1["label"], pred) - 147.4672) < 1e-3          # fm_loss_test.cc:35
    g = E.calc_grad(rcv1["offset"], lidx, rcv1["value"], rcv1["label"], w, pred)
    assert_close(g, refout["nov_grad"], what="grad", **GRAD_TOL)
    assert abs(float((g.astype(np.float64) ** 2).sum()) - 90.5817) < 1e-3  # fm_loss_test.cc:39


def test_fm_loss_hasv_golden(rcv1, refout):
    k = 5
    E = engine(V_dim=k)
    lidx = refout["loc_lidx"]
    U = len(refout["loc_keys"])
    W = refout["hasv_w"]
    w_pos = (np.arange(U) * (k + 1)).astype(np.int32)
    V_pos = w_pos + 1
    pred = E.predict(rcv1["offset"], lidx, rcv1["value"], W, w_pos, V_pos)
    assert_close(pred, refout["hasv_pred"], what="pred", **PRED_TOL)
    assert abs(E.evaluate(rcv1["label"], pred) - 330.628) < 1e-3           # fm_loss_test.cc:78
    g = E.calc_grad(rcv1["offset"], lidx, rcv1["value"], rcv1["label"], W, pred, w_pos, V_pos)
    assert_close(g, refout["hasv_grad"], what="grad", **GRAD_TOL)
    assert abs(float((g.astype(np.float64) ** 2).sum()) - 1.2378e3) < 1e-1  # fm_loss_test.cc:82


@pytest.mark.parametrize("V_dim,valued", [(0, True), (0, False), (3, False), (8, True), (64, False), (130, True)])
def test_loss_random_ragged_with_absent_V(V_dim, valued):
    rng = np.random.default_rng(100 + V_dim + int(valued))
    b = localized(rand_batch(rng, 300, 40, 700, valued))
    U = len(b["keys"])
    if V_dim == 0:
        W = (rng.standard_normal(U) * 0.1).astype(np.float32)
        w_pos = V_pos = None
    else:
        lens = np.where(rng.random(U) < 0.6, V_dim + 1, 1).astype(np.int32)   # V_pos = -1 holes
        w_pos, V_pos = O.get_pos(lens)
        W = (rng.standard_normal(int(lens.sum())) * 0.1).astype(np.float32)
    E = engine(V_dim=V_dim)
    init = rng.standard_normal(len(b["label"])).astype(np.float32) * 0.01
    ref_pred = O.fm_predict(V_dim, b["offset"], b["lidx"], b["value"], W, w_pos, V_pos)
    pred = E.predict(b["offset"], b["lidx"], b["value"], W, w_pos, V_pos)
    assert_close(pred, ref_pred, what="pred", **PRED_TOL)
    if V_dim == 0:
        # pred is accumulated into (spmv.h:127) -- only checkable without the clamp
        pred2 = E.predict(b["offset"], b["lidx"], b["value"], W, w_pos, V_pos, pred_init=init)
        assert_close(pred2, ref_pred + init, what="pred+=", **PRED_TOL)
    ref_g = O.fm_calc_grad(V_dim, b["offset"], b["lidx"], b["value"], b["label"], W, ref_pred, w_pos, V_pos)
    g = E.calc_grad(b["offset"], b["lidx"], b["value"], b["label"], W, ref_pred, w_pos, V_pos)
    assert_close(g, ref_g, what="grad", **GRAD_TOL)
    ginit = rng.standard_normal(len(W)).astype(np.float32)
    g2 = E.calc_grad(b["offset"], b["lidx"], b["value"], b["label"], W, ref_pred, w_pos, V_pos, grad_init=ginit)
    assert_close(g2, ref_g.astype(np.float64) + ginit, what="grad+=", rtol=1e-4, atol=1e-5)
    assert abs(E.evaluate(b["label"], ref_pred) - O.evaluate(b["label"], ref_pred)) <= 2e-5 * abs(O.evaluate(b["label"], ref_pred))


def test_v_dim0_is_not_clamped():
    # fm_loss.h:77 returns before the +-20 projection when V_dim == 0
    off = np.array([0, 2, 3], np.uint64)
    lidx = np.array([0, 1, 1], np.uint32)
    w = np.array([30.0, 25.0], np.float32)
    E = engine(V_dim=0)
    assert np.array_equal(E.predict(off, lidx, None, w), np.array([55.0, 25.0], np.float32))
    E2 = engine(V_dim=2)
    W = np.array([30.0, 0, 0, 25.0, 0, 0], np.float32)
    wp = np.array([0, 3], np.int32)
    assert np.array_equal(E2.predict(off, lidx, None, W, wp, wp + 1), np.array([20.0, 20.0], np.float32))


def test_auc_matches_reference_golden(refout):
    E = engine(V_dim=0)
    got = E.auc(refout["auc_label"], refout["auc_pred"])
    assert got == pytest.approx(float(refout["auc_value"]), rel=1e-6)
    assert E.auc(np.ones(7, np.float32), np.arange(7, dtype=np.float32)) == 1.0
    rng = np.random.default_rng(3)
    p = np.round(rng.standard_normal(4000), 1).astype(np.float32)   # many ties: stable order
    l = np.where(rng.random(4000) < 0.5, 1.0, 0.0).astype(np.float32)
    assert E.auc(l, p) == pytest.approx(O.auc(l, p), rel=1e-6)


# ----------------------------------------------------------------------------------------
# (A) Store/Updater: Pull / Push(kFeaCount) / Push(kGradient) bit-exact given identical inputs
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [0, 6, 16, 64])
def test_updater_bit_exact_given_oracle_gradients(V_dim):
    rng = np.random.default_rng(7 + V_dim)
    kw = dict(V_dim=V_dim, l1=0.4, l2=0.02, lr=0.3, V_lr=0.07, V_threshold=6, V_l2=0.05, V_init_scale=0.3,
              lr_beta=0.5, V_lr_beta=2.0, seed=99)
    M, E = O.Oracle(**kw), engine(**kw)
    seen = []
    for step in range(25):
        b = localized(rand_batch(rng, 64, 16, 260, step % 3 == 0))
        if step < 8:
            M.update_feacnt(b["keys"], b["cnt"])
            E.push_feacnt(b["keys"], b["cnt"])
        vals, lens = M.get(b["keys"])
        gv, gl = E.pull(b["keys"])
        assert np.array_equal(lens, gl), f"lens differ at step {step}"
        assert np.array_equal(vals, gv), f"pulled weights differ at step {step}"   # incl. InitV's rand_r stream
        if V_dim:
            w_pos, V_pos = O.get_pos(lens)
        else:
            w_pos = V_pos = None
        pred = O.fm_predict(V_dim, b["offset"], b["lidx"], b["value"], vals, w_pos, V_pos)
        g = O.fm_calc_grad(V_dim, b["offset"], b["lidx"], b["value"], b["label"], vals, pred, w_pos, V_pos)
        M.update_grad(b["keys"], g, lens)
        E.push_grad(b["keys"], g, lens)
        seen.append(b["keys"])
    keys = np.unique(np.concatenate(seen))
    scal, hasv, V, cg = E.read_entries(keys)
    oscal, ohasv, oV, ocg = oracle_state(M, keys)
    assert np.array_equal(hasv, ohasv)
    assert np.array_equal(scal, oscal)          # fea_cnt, w, sqrt_g, z bit-exact (FTRL)
    assert np.array_equal(V, oV) and np.array_equal(cg, ocg)   # AdaGrad + InitV bit-exact
    assert E.rng_state() == M.seed()
    st = E.table_stats()
    assert st["n_keys"] == M.size() and st["n_vrows"] == int((ohasv == 1).sum())
    if V_dim:
        assert (ohasv == 1).sum() > 10


def test_push_grad_checks_like_reference():
    E = engine(V_dim=4)
    keys = np.array([5, 9], np.uint64)
    with pytest.raises(capi.DfbError):      # CHECK_EQ(lens.size(), size)
        E.push_grad(keys, np.zeros(2, np.float32), np.array([1], np.int32))
    with pytest.raises(capi.DfbError):      # CHECK(e.V != nullptr): gradient for a key without V
        E.push_grad(keys, np.zeros(6, np.float32), np.array([5, 1], np.int32))
    with pytest.raises(capi.DfbError):      # CHECK_EQ(lens[i], V_dim+1)
        E.push_grad(keys, np.zeros(4, np.float32), np.array([3, 1], np.int32))
    E.push_grad(keys, np.zeros(2, np.float32), np.array([1, 1], np.int32))   # fine


def test_capacity_error_is_reported_not_fatal():
    E = capi.Engine(V_dim=0, table_capacity=64)
    with pytest.raises(capi.DfbError) as ei:
        E.pull(np.arange(1, 2000, dtype=np.uint64))
    assert ei.value.code == capi.DFB_ERR_CAPACITY


def test_param_errors_mirror_dmlc():
    with pytest.raises(capi.DfbError):
        capi.Engine(l1=1)                     # V_dim is required (sgd_param.h:104)
    with pytest.raises(capi.DfbError):
        capi.Engine(V_dim=2, lr=11)           # lr range [0, 10]
    E = capi.Engine(V_dim=2, foo="bar", batch_size=100)
    assert E.unknown_kwargs() == [("foo", "bar"), ("batch_size", "100")]


# ----------------------------------------------------------------------------------------
# (B) fused step vs the oracle's IterateData, whole trajectories
# ----------------------------------------------------------------------------------------
def run_both(kw, batches, epochs, force_generic=0, feacnt_epochs=1, val_every=0, scatter="sorted", **engine_kw):
    M = O.Oracle(**kw)
    E = engine(force_generic=force_generic, scatter=scatter, **engine_kw, **kw)
    t = 0
    for ep in range(epochs):
        for (o, l, i, v) in batches:
            b = localized((o, l, i, v))
            is_train = not (val_every and t % val_every == val_every - 1)
            push = ep < feacnt_epochs and is_train
            ref = M.sgd_step(o, i, v, l, is_train, push)
            pr, pred = E.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"] if push else None, is_train, want_pred=True)
            assert pr.nrows == ref[4]
            assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0]) + 1e-4, f"loss step {t}: {pr.loss} vs {ref[0]}"
            assert abs(pr.penalty - ref[1]) <= 1e-4 * abs(ref[1]) + 1e-5, f"penalty step {t}"
            t += 1
    return M, E


def compare_state(M, E, keys, tol=STATE_TOL):
    scal, hasv, V, cg = E.read_entries(keys)
    oscal, ohasv, oV, ocg = oracle_state(M, keys)
    assert np.array_equal(hasv, ohasv), "V allocation pattern differs"
    assert np.array_equal(scal[:, 0], oscal[:, 0])     # fea_cnt exact
    assert_close(scal[:, 1:], oscal[:, 1:], what="w/sqrt_g/z", **tol)
    assert_close(V, oV, what="V", **tol)
    assert_close(cg, ocg, what="cg", **tol)
    return ohasv


def test_fused_sgd_golden_trace_v0(rcv1, refout):
    # SGDLearner.Basic (sgd_learner_test.cc:9-49): 20 epochs over the 100-row fixture
    gold = refout["sgd_v0_trace"][:, 0]
    E = engine(V_dim=0, l1=1, l2=1, lr=1)
    for ep in range(20):
        pr = E.train_step(rcv1["offset"], refout["loc_lidx"], rcv1["value"], rcv1["label"], refout["loc_keys"],
                          refout["loc_cnt"] if ep == 0 else None, True)
        assert abs(pr.loss - float(gold[ep])) < 2e-4, f"epoch {ep}: {pr.loss} vs {gold[ep]}"


def test_fused_v8_trace_vs_reference(rcv1, refout):
    kw = parse_kwargs(refout["sgd_v8_kwargs"])
    E = engine(**kw)
    for ep in range(len(refout["sgd_v8_trace"])):
        pr = E.train_step(rcv1["offset"], refout["loc_lidx"], rcv1["value"], rcv1["label"], refout["loc_keys"],
                          refout["loc_cnt"] if ep == 0 else None, True)
        ref = refout["sgd_v8_trace"][ep]
        assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0])
        assert abs(pr.penalty - ref[1]) <= 1e-4 * abs(ref[1]) + 1e-6
    vals, lens = E.pull(refout["loc_keys"])
    assert np.array_equal(lens, refout["sgd_v8_final_lens"])      # same keys got a V row
    assert_close(vals, refout["sgd_v8_final_vals"], what="final [w,V]", **STATE_TOL)


@pytest.mark.parametrize("force_generic", [0, 1])
def test_fused_synthetic_trace_vs_reference(refout, force_generic):
    kw = parse_kwargs(refout["syn_kwargs"])   # V_dim = 16: fast path unless forced generic
    E = engine(force_generic=force_generic, **kw)
    batches = syn_batches(refout)
    t = 0
    for ep in range(3):
        for (o, l, i, v) in batches:
            b = localized((o, l, i, v))
            pr, pred = E.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"] if ep == 0 else None, True,
                                    want_pred=True)
            ref = refout["syn_trace"][t]
            assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0])
            assert abs(pr.penalty - ref[1]) <= 1e-4 * abs(ref[1]) + 1e-6
            # AUC: the reference's std::sort leaves the order of tied predictions unspecified
            # (bin_class_metric.h:44); ties keep row order here and in the oracle.
            assert pr.auc == pytest.approx(O.auc(l, pred), rel=1e-6)
            if len(np.unique(pred)) == len(pred):
                assert abs(pr.auc - ref[2]) <= 2e-3 * abs(ref[2]) + 0.5
            t += 1
    vals, lens = E.pull(refout["syn_keys"])
    assert np.array_equal(lens, refout["syn_final_lens"])
    assert_close(vals, refout["syn_final_vals"], what="final [w,V]", **STATE_TOL)


@pytest.mark.parametrize("V_dim,valued,force_generic,scatter",
                         [(0, True, 0, "sorted"), (5, True, 0, "sorted"), (8, False, 0, "sorted"), (8, True, 0, "atomic"),
                          (16, True, 0, "sorted"), (16, False, 0, "atomic"), (32, False, 0, "sorted"),
                          (64, True, 0, "sorted"), (64, True, 0, "atomic"), (64, False, 1, "sorted"),
                          (128, False, 0, "sorted"), (128, True, 0, "atomic")])
def test_fused_trajectory_vs_oracle(V_dim, valued, force_generic, scatter):
    rng = np.random.default_rng(1000 + V_dim)
    kw = dict(V_dim=V_dim, l1=0.3, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=4, V_l2=0.02, V_init_scale=0.2, seed=5)
    batches = [rand_batch(rng, 128, 30, 400, valued and j % 2 == 0) for j in range(5)]
    M, E = run_both(kw, batches, epochs=4, force_generic=force_generic, val_every=4, scatter=scatter)
    keys = np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b in batches]))
    ohasv = compare_state(M, E, keys)
    assert E.rng_state() == M.seed()
    if V_dim:
        assert (ohasv == 1).sum() > 10


def test_very_hot_keys_prereduced_in_chunks_vs_oracle():
    """occurrence lists longer than hot_split are cut into chunks reduced by separate warps (k_hot_reduce) and the
    partials added in chunk order: a feature present in EVERY row (the Criteo case), a threshold low enough
    that the ~400-occurrence keys take the path too, binary and valued batches, the fused and the sharded kernel"""
    rng = np.random.default_rng(99)
    kw = dict(V_dim=16, l1=0.01, l2=0.01, lr=0.05, V_lr=0.02, V_threshold=0, V_l2=0.02, V_init_scale=0.1, seed=8)
    batches = []
    for valued in (False, True, False):
        b = rand_batch(rng, 3000, 12, 25, valued, min_nnz=4)
        b[2][b[0][:-1].astype(np.int64)] = (np.array([77], np.uint64) * np.uint64(0x9E3779B97F4A7C15))[0]     # first nnz of every row: one feature
        batches.append(b)
    M, E = run_both(kw, batches, epochs=2, val_every=0, hot_split=100)
    keys = np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b in batches]))
    compare_state(M, E, keys, tol=dict(rtol=2e-3, atol=2e-5))
    # bit-reproducible, and the default threshold (the same lists reduced by one warp each) agrees within rounding
    E2 = run_both(kw, batches, epochs=2, val_every=0, hot_split=100)[1]
    for a, b in zip(E.read_entries(keys), E2.read_entries(keys)):
        assert np.array_equal(a, b)
    E3 = run_both(kw, batches, epochs=2, val_every=0, hot_split=0)[1]
    for a, b in zip(E.read_entries(keys), E3.read_entries(keys)):
        assert_close(a, b, what="pre-reduced vs one warp", rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("V_dim,valued", [(16, True), (64, False), (128, True)])
def test_hot_keys_vs_oracle(V_dim, valued):
    # a skewed batch: 25 features shared by 700 rows -> ~400 occurrences per key, far above the
    # threshold at which a key's gradient is reduced by a whole warp instead of one lane group
    rng = np.random.default_rng(4242 + V_dim)
    kw = dict(V_dim=V_dim, l1=0.01, l2=0.01, lr=0.05, V_lr=0.02, V_threshold=0, V_l2=0.02, V_init_scale=0.1, seed=8)
    batches = [rand_batch(rng, 700, 30, 25, valued, min_nnz=5) for _ in range(3)]
    # plus a few cold keys so that short and long lists share warps
    for b in batches:
        b[2][::17] = rng.integers(10 ** 6, 10 ** 7, len(b[2][::17])).astype(np.uint64)
    M, E = run_both(kw, batches, epochs=3, val_every=0)
    keys = np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b in batches]))
    compare_state(M, E, keys, tol=dict(rtol=2e-3, atol=2e-5))
    R = engine(**kw)
    for ep in range(3):
        for (o, l, i, v) in batches:
            R.train_step_raw(o, i, v, l, push_cnt=(ep == 0), is_train=True)
    for a, b in zip(R.read_entries(keys), E.read_entries(keys)):
        assert np.array_equal(a, b)        # GPU-localized and host-localized paths are bit-identical


def test_edge_cases_empty_rows_and_batches():
    kw = dict(V_dim=8, l1=0.0, l2=0.0, lr=0.1, V_threshold=0, seed=1)
    M, E = O.Oracle(**kw), engine(**kw)
    # a batch whose rows are all empty, and a batch with zero rows
    off = np.zeros(5, np.uint64)
    lab = np.array([1, -1, 1, -1], np.float32)
    pr = E.train_step(off, np.zeros(0, np.uint32), None, lab, np.zeros(0, np.uint64), None, True)
    ref = M.sgd_step(off, np.zeros(0, np.uint64), None, lab, True, False)
    assert pr.nrows == 4 and abs(pr.loss - ref[0]) < 1e-5
    pr = E.train_step(np.zeros(1, np.uint64), np.zeros(0, np.uint32), None, np.zeros(0, np.float32),
                      np.zeros(0, np.uint64), None, True)
    assert pr.nrows == 0 and pr.loss == 0
    # one very long row (gisette-like) next to empty rows, duplicate ids inside a row
    rng = np.random.default_rng(2)
    ids = rng.integers(0, 50, 3000).astype(np.uint64)
    off = np.array([0, 0, 3000, 3000, 3001], np.uint64)
    idx = np.concatenate([ids, [7]]).astype(np.uint64)
    val = rng.random(3001).astype(np.float32) * 0.02
    lab = np.array([1, -1, 1, 1], np.float32)
    for t in range(4):
        b = localized((off, lab, idx, val))
        ref = M.sgd_step(off, idx, val, lab, True, t == 0)
        pr = E.train_step(off, b["lidx"], val, lab, b["keys"], b["cnt"] if t == 0 else None, True)
        assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0]) + 1e-5
    compare_state(M, E, localized((off, lab, idx, val))["keys"])


@pytest.mark.parametrize("V_dim,valued", [(16, True), (64, False), (128, True)])
def test_long_rows_cta_per_row_vs_oracle(V_dim, valued):
    """gisette-shaped examples (5000 nonzeros) next to rows just below / at / above long_row_nnz, short and empty
    ones: rows of >= long_row_nnz nonzeros are walked by a whole CTA (k_fm_long), the others by one warp
    (k_fm_fast) -- trajectory and predictions against the oracle, and against the engine with the long path off"""
    rng = np.random.default_rng(9)
    lens = np.array([5000, 0, 1023, 1024, 1025, 40, 4999, 7, 2048, 0, 3], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    n = int(off[-1])
    idx = rng.integers(0, 5000, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    val = (rng.random(n).astype(np.float32) * 0.05) if valued else None
    lab = np.where(rng.random(len(lens)) < 0.5, 1.0, -1.0).astype(np.float32)
    kw = dict(V_dim=V_dim, l1=0.01, l2=0.01, lr=0.05, V_lr=0.02, V_threshold=0, V_init_scale=0.01 if valued else 0.002,
              seed=5)
    M = O.Oracle(**kw)
    E = engine(**kw)
    W = engine(long_row_nnz=0, **kw)
    for t in range(4):
        is_train = t != 2
        ref = M.sgd_step(off, idx, val, lab, is_train, t == 0)
        pr, pred = E.train_step_raw(off, idx, val, lab, push_cnt=(t == 0), is_train=is_train, want_pred=True)
        prw, predw = W.train_step_raw(off, idx, val, lab, push_cnt=(t == 0), is_train=is_train, want_pred=True)
        assert abs(pr.loss - ref[0]) <= 1e-4 * abs(ref[0]) + 1e-5, f"step {t}: {pr.loss} vs {ref[0]}"
        assert_close(pred, predw, what=f"CTA-per-row vs warp-per-row pred, step {t}", rtol=1e-4, atol=1e-5)
    keys = localized((off, lab, idx, val))["keys"]
    compare_state(M, E, keys)
    compare_state(M, W, keys)


def test_validation_step_does_not_update():
    rng = np.random.default_rng(11)
    kw = dict(V_dim=16, l1=0.01, lr=0.1, V_threshold=0, seed=4)
    E = engine(**kw)
    b = localized(rand_batch(rng, 100, 20, 300, False))
    E.train_step(b["offset"], b["lidx"], None, b["label"], b["keys"], b["cnt"], True)
    before = E.read_entries(b["keys"])
    pr1, p1 = E.train_step(b["offset"], b["lidx"], None, b["label"], b["keys"], None, False, want_pred=True)
    pr2, p2 = E.train_step(b["offset"], b["lidx"], None, b["label"], b["keys"], None, False, want_pred=True)
    after = E.read_entries(b["keys"])
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    assert np.array_equal(p1, p2) and pr1.loss == pr2.loss     # forward is deterministic


def test_sorted_scatter_is_bit_reproducible():
    # the sorted reduction sums each key's contributions in row order: two runs are bit-identical,
    # and hot keys (many occurrences) are reduced in the reference's order (spmm.h:140-156)
    rng = np.random.default_rng(21)
    kw = dict(V_dim=32, l1=0.01, lr=0.1, V_threshold=0, seed=9, scatter="sorted")
    batches = [localized(rand_batch(rng, 512, 40, 60, j % 2 == 0)) for j in range(4)]   # 60 ids: heavy reuse
    states = []
    for rep in range(2):
        E = engine(**kw)
        for ep in range(3):
            for b in batches:
                E.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], b["cnt"] if ep == 0 else None, True)
        keys = np.unique(np.concatenate([b["keys"] for b in batches]))
        states.append(E.read_entries(keys))
    for a, b in zip(*states):
        assert np.array_equal(a, b)


def test_checkpoint_roundtrip_and_resume():
    # Updater::Save/Load (updater.h:40-47): restore into a fresh engine, then continue training --
    # bit-identical to the uninterrupted run (sorted path), incl. the InitV random stream
    rng = np.random.default_rng(31)
    kw = dict(V_dim=16, l1=0.05, lr=0.2, V_lr=0.1, V_threshold=1, V_init_scale=0.2, seed=6)
    batches = [localized(rand_batch(rng, 200, 25, 600, j % 2 == 0)) for j in range(6)]

    def step(E, b, first):
        return E.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], b["cnt"] if first else None, True)

    A = engine(**kw)
    for b in batches[:3]:
        step(A, b, True)
    blob = A.snapshot(save_aux=True)
    B = engine(**kw)
    assert B.restore(blob) is True
    assert B.table_stats()["n_keys"] == A.table_stats()["n_keys"] and B.rng_state() == A.rng_state()
    keys = np.unique(np.concatenate([b["keys"] for b in batches]))
    for x, y in zip(A.read_entries(keys), B.read_entries(keys)):
        assert np.array_equal(x, y)
    for b in batches[3:]:
        pa, pb = step(A, b, True), step(B, b, True)
        assert pa.loss == pb.loss
    for x, y in zip(A.read_entries(keys), B.read_entries(keys)):
        assert np.array_equal(x, y)
    assert A.snapshot() == B.snapshot()              # deterministic byte format (ascending keys)
    # a snapshot without aux data predicts but cannot train (CHECK(has_aux_), sgd_updater.cc:75)
    C2 = engine(**kw)
    assert C2.restore(A.snapshot(save_aux=False)) is False
    b = batches[0]
    pv = C2.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, False)
    pa = A.train_step(b["offset"], b["lidx"], b["value"], b["label"], b["keys"], None, False)
    assert pv.loss == pa.loss
    with pytest.raises(capi.DfbError):
        step(C2, b, False)
    with pytest.raises(capi.DfbError):                # restore needs an empty table / same V_dim
        A.restore(blob)
    with pytest.raises(capi.DfbError):
        engine(**dict(kw, V_dim=8)).restore(blob)


def test_async_pipeline_equals_sync():
    rng = np.random.default_rng(12)
    kw = dict(V_dim=32, l1=0.05, lr=0.1, V_threshold=1, seed=4)
    batches = [localized(rand_batch(rng, 200, 25, 800, False)) for _ in range(6)]
    A, S = engine(**kw), engine(**kw)
    for b in batches:
        S.train_step(b["offset"], b["lidx"], None, b["label"], b["keys"], b["cnt"], True)
    for b in batches:
        A.train_step_async(len(b["label"]), b["offset"], b["lidx"], None, b["label"], b["keys"], len(b["keys"]),
                           b["cnt"], True)
    pr = A.read_progress()
    assert pr.nrows == 200 * 6
    keys = np.unique(np.concatenate([b["keys"] for b in batches]))
    sa, ss = A.read_entries(keys), S.read_entries(keys)
    assert np.array_equal(sa[1], ss[1])
    assert_close(sa[0], ss[0], what="scal", **STATE_TOL)
    assert_close(sa[2], ss[2], what="V", **STATE_TOL)
    assert A.launch_count() > 0


# ----------------------------------------------------------------------------------------
# full-size (BASELINE.json synthetic shape): size-independent properties
# ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [16, 64])
def test_full_size_properties(V_dim):
    B, NNZ = 65536, 100
    rng = np.random.default_rng(77)
    ids = rng.integers(0, 10 ** 9, B * NNZ).astype(np.uint64)
    off = (np.arange(B + 1, dtype=np.uint64) * np.uint64(NNZ))
    lab = np.where(rng.random(B) < 0.3, 1.0, -1.0).astype(np.float32)
    # vectorised localize (numpy): reversed keys, sorted unique, ranks
    rk = O.reverse_bytes_np(ids)
    keys, lidx, cnt = np.unique(rk, return_inverse=True, return_counts=True)
    lidx = lidx.astype(np.uint32)
    cnt = cnt.astype(np.float32)
    kw = dict(V_dim=V_dim, l1=0.0, l2=0.0, lr=0.05, V_lr=0.05, V_threshold=0, V_init_scale=0.05, seed=2,
              table_capacity=1 << 23)
    E = capi.Engine(**kw)
    G = capi.Engine(force_generic=1, **kw)
    for eng in (E, G):   # two steps: the first creates w (V rows appear on the 0 -> nonzero transition)
        eng.train_step(off, lidx, None, lab, keys, cnt, True)
        eng.train_step(off, lidx, None, lab, keys, None, True)
    st = E.table_stats()
    assert st["n_keys"] == len(keys) and st["n_vrows"] == len(keys)   # every key has a V row now
    assert E.rng_state() == G.rng_state()
    prE, pE = E.train_step(off, lidx, None, lab, keys, None, False, want_pred=True)
    prG, pG = G.train_step(off, lidx, None, lab, keys, None, False, want_pred=True)
    # 1. fast kernel == independent generic kernel
    assert_close(pE, pG, what="fast vs generic pred", rtol=1e-4, atol=1e-4)
    assert abs(prE.loss - prG.loss) <= 1e-4 * abs(prG.loss)
    # 2. a sample of rows against the oracle through the API-faithful pull
    rows = rng.choice(B, 200, replace=False)
    sub_idx = np.concatenate([ids[r * NNZ:(r + 1) * NNZ] for r in rows])
    sub_off = (np.arange(len(rows) + 1, dtype=np.uint64) * np.uint64(NNZ))
    sl, sk, _ = O.localize(sub_off, sub_idx)
    vals, lens = E.pull(sk)
    w_pos, V_pos = O.get_pos(lens)
    ref = O.fm_predict(V_dim, sub_off, sl, None, vals, w_pos, V_pos)
    assert_close(pE[rows], ref, what="sampled rows vs oracle", **PRED_TOL)
    # 3. checksum: sum_keys grad_w == sum_rows p_i * nnz_i  <=> after one more FTRL step with l1=l2=0
    #    the table still holds exactly len(keys) keys and AUC is in [0.5, 1] * B
    assert 0.5 * B <= prE.auc <= B


def test_full_size_training_steps_vs_oracle():
    """BASELINE.json's synthetic shape (65536 rows x 100 nnz, raw uint64 ids) through the fused raw-id step -- GPU
    localizer, lookup/insert, InitV, forward, per-key gradient reduce, FTRL/AdaGrad -- against the oracle running the
    SAME three minibatches (about 12 s of CPU per step): loss and penalty per step, and the full state of a 4000-key
    sample (plus the 200 most frequent keys) after the third update.  V_dim = 16 keeps the oracle's share bearable."""
    B, NNZ, k = 65536, 100, 16
    rng = np.random.default_rng(78)
    off = (np.arange(B + 1, dtype=np.uint64) * np.uint64(NNZ))
    kw = dict(V_dim=k, l1=0.02, l2=0.01, lr=0.05, V_lr=0.05, V_l2=0.01, V_threshold=2, V_init_scale=0.05, seed=2)
    M = O.Oracle(**kw)
    E = capi.Engine(table_capacity=1 << 25, **kw)
    seen = []
    for t in range(3):
        # a skewed head (hot keys, V rows appear after two counts) over a uniform tail (mostly new keys every step)
        hot = rng.zipf(1.3, B * NNZ) % 5000
        ids = np.where(rng.random(B * NNZ) < 0.3, hot, rng.integers(0, 3 * 10 ** 7, B * NNZ)).astype(np.uint64)
        ids *= np.uint64(0x9E3779B97F4A7C15)
        lab = np.where(rng.random(B) < 0.3, 1.0, -1.0).astype(np.float32)
        # the oracle's step, with its first two calls (Update(kFeaCount), Get: sgd_learner.cc:214-217, :177) made here so
        # that the pulled weights are at hand for a float64 penalty
        keys_t, cnt_t = np.unique(O.reverse_bytes_np(ids), return_counts=True)
        M.update_feacnt(keys_t, cnt_t.astype(np.float32))
        vals, lens = M.get(keys_t)
        w_pos, _ = O.get_pos(lens)
        w64 = vals[w_pos].astype(np.float64)
        pen64 = (kw["l1"] * np.abs(w64).sum() + 0.5 * kw["l2"] * (w64 ** 2).sum()
                 + 0.5 * kw["V_l2"] * ((vals.astype(np.float64) ** 2).sum() - (w64 ** 2).sum()))
        ref = M.sgd_step(off, ids, None, lab, True, False)
        pr = E.train_step_raw(off, ids, None, lab, push_cnt=True, is_train=True)
        assert pr.nrows == ref[4] == B
        # the reference sums the 65536 row losses and the ~5 M penalty terms sequentially in float32 (loss.h:57-66,
        # sgd_learner.cc:249-273): at this size the running sums themselves are off by a few 1e-4 (loss: step 0, an
        # empty model, is exactly 65536 ln 2 = 45426.1 here, 45437.3 there) to ~1e-2 (penalty: terms of 4e-5 added to
        # a sum near 200, half an ulp each); the engine accumulates in double, so the penalty is checked tightly
        # against the float64 sum over the weights the oracle pulled, and loosely against the oracle's float sum
        assert abs(pr.loss - ref[0]) <= 1e-3 * abs(ref[0]), f"loss step {t}: {pr.loss} vs {ref[0]}"
        assert abs(pr.penalty - pen64) <= 1e-5 * abs(pen64) + 1e-6, f"penalty step {t}: {pr.penalty} vs {pen64}"
        assert abs(pr.penalty - ref[1]) <= 3e-2 * abs(ref[1]) + 1e-5, f"penalty step {t}: {pr.penalty} vs {ref[1]}"
        seen.append(ids)
    assert E.table_stats()["n_keys"] == M.size()
    assert E.rng_state() == M.seed()
    allk, cnt = np.unique(O.reverse_bytes_np(np.concatenate(seen)), return_counts=True)
    sample = np.unique(np.concatenate([rng.choice(allk, 4000, replace=False), allk[np.argsort(cnt)[-200:]]]))
    hasv = compare_state(M, E, sample)
    assert (hasv > 0).sum() > 200 and (hasv <= 0).sum() > 200      # both kinds of keys were compared
