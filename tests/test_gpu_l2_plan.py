"""The L2 plan of the single-GPU training step (engine kwarg l2_hints): when the table rows a step touches exceed the L2,
the fused update keeps p*XV / p evict_last, streams the [V|cg] rows evict_first (k_bwd_update<K, VAL, true, 0, true>,
k_hot_reduce under the hint) and then drops p*XV / p from L2 with discard.global.L2 (k_l2_discard).  Cache policies
must not change a single bit: with the plan on, the model equals the one trained with l2_hints=0 bit for bit, and
the oracle within the suite's tolerances.

The batch shapes are computed from the device's L2 and the rule of step_dev (engine.cu): the plan is on when
u_bound * rs * 4 bytes > L2, where rs = 2 V_dim floats and u_bound is the batch's nnz for a raw step (capped at
2^id_bits when id_bits < 40).  The plan adds exactly one launch (k_l2_discard) to a training step, which is how the
tests see that it ran -- and that one nnz less keeps it off."""
import numpy as np
import pytest

from oracle import oracle as O
from util import assert_close, localized, oracle_state

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
STATE_TOL = dict(rtol=1e-3, atol=1e-5)
KW = dict(l1=0.01, l2=0.01, lr=0.05, V_lr=0.05, V_l2=0.01, V_threshold=1, V_init_scale=0.05, seed=3)
LONG_ROWS = (1024, 1100, 1500)        # >= long_row_nnz (1024): k_fm_long's rows


def l2_bytes():
    return torch.cuda.get_device_properties(0).L2_cache_size


def plan_threshold_nnz(K):
    """the largest raw batch (nnz) whose rows still fit in L2: one nnz more turns the plan on"""
    return l2_bytes() // (2 * K * 4)


def plan_on(nnz, K):
    return nnz * 2 * K * 4 > l2_bytes()


def plan_batch(rng, nnz, pool, valued, hot_id):
    """exactly nnz ids: rows of 0..59 ids, three rows of >= long_row_nnz, and hot_id as the first id of every third row
    (thousands of occurrences: far above hot_split = 256, so k_hot_reduce pre-reduces it)"""
    rest = nnz - sum(LONG_ROWS)
    lens = rng.integers(0, 60, rest // 25 + 64)
    c = np.cumsum(lens)
    k = int(np.searchsorted(c, rest))
    lens = lens[:k + 1].copy()
    lens[-1] -= int(c[k]) - rest
    for j, n in enumerate(LONG_ROWS):
        lens = np.insert(lens, (j + 1) * len(lens) // 4, n)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(U64)
    assert int(off[-1]) == nnz
    ids = pool[rng.integers(0, len(pool), nnz)]
    starts = off[:-1][lens > 0][::3].astype(np.int64)
    ids[starts] = hot_id
    val = (rng.random(nnz).astype(np.float32) * 0.5) if valued else None
    lab = np.where(rng.random(len(lens)) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, lab, ids, val


def run(E, seq):
    out = []
    for (o, l, i, v), is_train in seq:
        pr = E.train_step_raw(o, i, v, l, push_cnt=is_train, is_train=is_train)
        out.append((pr.loss, pr.penalty, pr.auc, pr.nrows, pr.new_keys, pr.new_vrows))
    return out


@pytest.mark.parametrize("K,valued,above", [(8, False, True), (8, True, True), (16, False, True), (16, True, True),
                                            (32, False, True), (32, True, True), (64, False, True), (64, True, True),
                                            (128, False, True), (128, True, True), (64, False, False)])
def test_l2_plan_bit_identical_and_vs_oracle(K, valued, above):
    """three training steps, a validation step, then a training batch with fewer rows than the one before it"""
    rng = np.random.default_rng(K * 2 + valued + 10 * above)
    thr = plan_threshold_nnz(K)
    nnz = thr + 1 if above else thr
    pool = np.unique(rng.integers(0, 1 << 40, nnz // 16, dtype=U64))
    hot = pool[0]
    seq = [(plan_batch(rng, nnz, pool, valued and j != 1, hot), True) for j in range(3)]
    seq.append((plan_batch(rng, nnz, pool, valued, hot), False))
    small = plan_batch(rng, nnz * 3 // 5, pool, valued, hot)
    assert len(small[1]) < len(seq[-1][0][1])
    seq.append((small, True))
    n_plan = sum(plan_on(int(b[0][-1]), K) for b, tr in seq if tr)
    assert n_plan == (3 if above else 0) + plan_on(int(small[0][-1]), K)

    kw = dict(V_dim=K, table_capacity=1 << 20, **KW)
    H = capi.Engine(l2_hints=1, **kw)
    N = capi.Engine(l2_hints=0, **kw)
    M = O.Oracle(V_dim=K, **KW)
    lc_h, lc_n = H.launch_count(), N.launch_count()
    prog_h, prog_n = run(H, seq), run(N, seq)
    assert (H.launch_count() - lc_h) - (N.launch_count() - lc_n) == n_plan      # one k_l2_discard per planned step
    assert prog_h == prog_n
    for t, (((o, l, i, v), is_train), ph) in enumerate(zip(seq, prog_h)):
        ref = M.sgd_step(o, i, v, l, is_train, is_train)
        assert ph[3] == ref[4]
        # the oracle sums its row losses sequentially in float32: off by up to ~1e-3 at these sizes (see
        # test_full_size_training_steps_vs_oracle); the engine sums in double
        assert abs(ph[0] - ref[0]) <= 1e-3 * abs(ref[0]), f"loss step {t}: {ph[0]} vs {ref[0]}"
        assert abs(ph[1] - ref[1]) <= 3e-2 * abs(ref[1]) + 1e-5, f"penalty step {t}: {ph[1]} vs {ref[1]}"
    keys = np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b, _ in seq]))
    eh = H.read_entries(keys)
    for a, b in zip(eh, N.read_entries(keys)):
        assert np.array_equal(a, b)
    assert H.rng_state() == N.rng_state() == M.seed()
    scal, hasv, V, cg = eh
    oscal, ohasv, oV, ocg = oracle_state(M, keys)
    assert np.array_equal(hasv, ohasv) and (hasv == 1).sum() > len(keys) // 4
    assert np.array_equal(scal[:, 0], oscal[:, 0])
    assert_close(scal[:, 1:], oscal[:, 1:], what="w/sqrt_g/z", **STATE_TOL)
    assert_close(V, oV, what="V", **STATE_TOL)
    assert_close(cg, ocg, what="cg", **STATE_TOL)


def auc_np(label, pred):
    """BinClassMetric::AUC (src/loss/bin_class_metric.h:35-56 of the reference) in float64: a stable sort by prediction"""
    pos = label[np.argsort(pred, kind="stable")] > 0
    n, tp = len(pred), int(pos.sum())
    if tp == 0 or tp == n:
        return 1.0
    area = float(np.cumsum(pos)[~pos].sum()) / (float(tp) * float(n - tp))
    return (1.0 - area if area < 0.5 else area) * n


def test_flagship_config_full_size():
    """bench.py's flagship engine (id_bits=30, V_dim 64, --hyper allV, overlap_auc=1) on two 65536 x 100 batches of ids
    below 1e9: 32-bit sort keys, the L2 plan on, the pulled view not kept in L2.  Three device-resident raw steps equal
    the host-localized steps of an engine without L2 hints bit for bit; the validation AUC equals a float64 AUC of
    the returned predictions.  The two engines take about 16 GB of HBM."""
    B, NNZ, K = 65536, 100, 64
    rng = np.random.default_rng(2024)
    off = np.arange(B + 1, dtype=U64) * U64(NNZ)
    batches = [(off, np.where(rng.random(B) < 0.3, 1.0, -1.0).astype(np.float32),
                rng.integers(0, 10 ** 9, B * NNZ).astype(U64), None) for _ in range(2)]
    assert plan_on(B * NNZ, K) and B * NNZ * 8 > l2_bytes() // 2
    allv = dict(V_dim=K, l1=0.0, l2=0.0, lr=0.01, lr_beta=1.0, V_l2=0.01, V_lr=0.01, V_lr_beta=1.0, V_init_scale=0.01,
                V_threshold=0, seed=0)
    cap = 14_000_000          # > the ~12.96 M distinct ids of both batches
    E = capi.Engine(table_capacity=cap, V_capacity=cap, id_bits=30, overlap_auc=1, **allv)
    T = capi.Engine(table_capacity=cap, V_capacity=cap, l2_hints=0, **allv)
    loc = []
    for (o, l, i, v) in batches:     # Localizer::Compact, vectorised
        keys, lidx, cnt = np.unique(O.reverse_bytes_np(i), return_inverse=True, return_counts=True)
        loc.append((lidx.astype(np.uint32), keys, cnt.astype(np.float32)))
    dev = torch.device("cuda", 0)
    devb = [(torch.from_numpy(o.view(np.int64)).to(dev), torch.from_numpy(l).to(dev),
             torch.from_numpy(i.view(np.int64)).to(dev)) for (o, l, i, v) in batches]
    torch.cuda.synchronize()
    for t, j in enumerate((0, 1, 0)):
        push = t < 2
        do, dl, di = devb[j]
        E.train_step_raw_dev(B, B * NNZ, do, di, None, dl, push, True)
        pe = E.read_progress()
        o, l, i, _ = batches[j]
        lidx, keys, cnt = loc[j]
        pt = T.train_step(o, lidx, None, l, keys, cnt if push else None, True)
        assert pe.loss == pt.loss and pe.penalty == pt.penalty and pe.auc == pt.auc, f"step {t}"
        assert (pe.nrows, pe.new_keys, pe.new_vrows) == (pt.nrows, pt.new_keys, pt.new_vrows), f"step {t}"
    allk, cnt = np.unique(O.reverse_bytes_np(np.concatenate([b[2] for b in batches])), return_counts=True)
    sample = np.unique(np.concatenate([rng.choice(allk, 20000, replace=False), allk[np.argsort(cnt, kind="stable")[-200:]]]))
    for a, b in zip(E.read_entries(sample), T.read_entries(sample)):
        assert np.array_equal(a, b)
    assert E.rng_state() == T.rng_state() and E.table_stats() == T.table_stats()
    o, l, i, _ = batches[1]
    pe, pred = E.train_step_raw(o, i, None, l, is_train=False, want_pred=True)
    pt, predt = T.train_step(o, loc[1][0], None, l, loc[1][1], None, False, want_pred=True)
    assert np.array_equal(pred, predt) and pe.loss == pt.loss
    assert pe.auc == np.float32(auc_np(l, pred))
    assert 0.5 * B <= pe.auc <= B
