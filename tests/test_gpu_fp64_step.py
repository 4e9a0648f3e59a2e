"""Full-size training steps against the float64 one-step reference (fp64_step.py): every key a step touches, compared
with an independent float64 statement of the step started from the exact state the engine held before it, within
error bounds derived for that one step (no flat tolerance).  Keys outside the batch -- a sample of at least 100 k of
the keys earlier batches brought, their hottest keys among them, and ids the table never saw -- must not change by a
bit.  Predictions are checked where a step returns them, and the AUC of the returned predictions against float64.

Cases: bench.py's flagship (synthetic 65536 x 100, ids below 1e9, id_bits = 30, V_dim 64, allV) through pass 0 with the
count push (cold inserts, ~6.5 M InitV rows per step) and pass 1 without it (the lookup-free raw step, checked to run
without k_lookup), a validation and a predict step, and a batch of only new ids; V_dim 0 ... 128 binary and valued above
the L2 bound with a hot id and long rows; criteo39 at every sweep point; gisette; rcv1; both sides of the L2 plan's
threshold.  Then the sharpness check: every deliberately wrong variant of the reference rejects the engine's step that
the true reference accepts.  Each case prints its largest error-to-bound ratio and its count of ambiguous keys."""
import argparse
import time

import numpy as np
import pytest

import bench
import fp64_step as F
import test_gpu_id_range as idr
import test_gpu_l2_plan as l2p
import test_gpu_lookup_free_step as lf

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
N_OUTSIDE = 100_000


def bench_args(**kw):
    a = dict(workload="synthetic", batch=65536, nnz=100, id_space=10 ** 9, vdim=64, hyper="allV")
    a.update(kw)
    return argparse.Namespace(**a)


def bench_engine(args, cap, **extra):
    """the engine run_single builds for args (bench.py), with capacity cap"""
    id_bits = {"synthetic": int(np.ceil(np.log2(float(args.id_space)))), "gisette": 13, "rcv1": 16}.get(args.workload, 64)
    return capi.Engine(device=0, table_capacity=cap, V_capacity=cap, id_bits=min(id_bits, 64), overlap_auc=1,
                       **extra, **bench.hyper(args))


class Run:
    """an engine and the keys its batches brought so far (for the sample outside each step's batch)"""

    def __init__(self, E, hp, hot_chunk=256, amb_frac=F.AMB_FRAC):
        self.E, self.hp, self.hot_chunk, self.amb_frac = E, hp, hot_chunk, amb_frac
        self.seen, self.seen_cnt = np.zeros(0, U64), np.zeros(0, np.int64)
        self.rng = np.random.default_rng(99)
        self.reports = []

    def outside(self, keys):
        rest = np.setdiff1d(self.seen, keys, assume_unique=True)
        cnt = self.seen_cnt[np.searchsorted(self.seen, rest)] if len(rest) else np.zeros(0, np.int64)
        pick = [self.rng.choice(rest, min(N_OUTSIDE, len(rest)), replace=False) if len(rest) else rest,
                rest[np.argsort(cnt, kind="stable")[-1000:]],
                np.setdiff1d(self.rng.integers(1, 1 << 62, 2000).astype(U64), keys)]          # never seen
        return np.unique(np.concatenate(pick))

    def step(self, b, kind, push=False, dev=None, mutants=()):
        """one step of the engine (kind: train_dev / train_pred / val / predict), held to the reference"""
        E = self.E
        o, l, i, v = b
        keys, _, cnt = F.batch_keys(i)
        pre = E.read_entries(keys)
        out = self.outside(keys)
        out_pre = E.read_entries(out)
        seed0, st0 = E.rng_state(), E.table_stats()
        pred = None
        t0 = time.perf_counter()
        if kind == "train_dev":
            do, dl, di, dv = dev
            E.train_step_raw_dev(len(l), len(i), do, di, dv, dl, push, True)
            pr = E.read_progress()
        elif kind == "train_pred":
            pr, pred = E.train_step_raw(o, i, v, l, push_cnt=push, is_train=True, want_pred=True)
        elif kind == "val":
            pr, pred = E.train_step_raw(o, i, v, l, push_cnt=False, is_train=False, want_pred=True)
        else:
            pr, pred = E.predict_raw(o, i, v, l)
        t_step = time.perf_counter() - t0
        post = E.read_entries(keys)
        st1 = E.table_stats()
        obs = dict(loss=pr.loss, penalty=pr.penalty, nrows=pr.nrows, new_keys=pr.new_keys, new_vrows=pr.new_vrows,
                   n_keys_delta=st1["n_keys"] - st0["n_keys"], n_vrows_delta=st1["n_vrows"] - st0["n_vrows"],
                   rng_after=E.rng_state(), pred=pred, auc=pr.auc, label=l)
        mode = {"train_dev": "train", "train_pred": "train"}.get(kind, kind)
        t0 = time.perf_counter()
        ref = F.Reference(b, self.hp, pre, seed0, push, mode, "cuda", hot_chunk=self.hot_chunk, val_inserts=False)
        R = F.check(ref, pre, post, obs, what=f"{kind} push={push}", pen_partial=F.pen_partial_engine,
                    amb_frac=self.amb_frac)
        t_ref = time.perf_counter() - t0
        print(f"{R.summary()}; engine {t_step:.2f} s, reference + comparison {t_ref:.1f} s, keys {len(keys)}")
        R.assert_ok()
        F.assert_unchanged(out_pre, E.read_entries(out), out, f"{kind} push={push}")
        for m in mutants:
            Rm = F.check(F.Reference(b, self.hp, pre, seed0, push, mode, "cuda", mutant=m, hot_chunk=self.hot_chunk,
                                     val_inserts=False),
                         pre, post, obs, what=m, pen_partial=F.pen_partial_engine)
            assert not Rm.ok(), f"the {m} variant of the reference accepts the engine's step: {Rm.summary()}"
        if mode != "predict":
            allk = np.concatenate([self.seen, keys])
            allc = np.concatenate([self.seen_cnt, cnt])
            self.seen, inv = np.unique(allk, return_inverse=True)
            self.seen_cnt = np.zeros(len(self.seen), np.int64)
            np.add.at(self.seen_cnt, inv, allc)
        self.reports.append(R)
        del ref
        torch.cuda.empty_cache()
        return R


def peak_gb():
    return torch.cuda.max_memory_allocated() / 2 ** 30


def test_flagship_as_bench_runs_it():
    """bench.py's engine and batches: pass 0 with the count push, pass 1 without it (lookup-free), a validation and a
    predict step, then a batch of only new ids (lookup-free inserts, no V rows)"""
    args = bench_args()
    batches = [bench.gen_raw_batch(args, s) for s in (1, 2)]
    cold = bench.gen_raw_batch(args, 3)
    cold = (cold[0], cold[1], U64(10 ** 9) + cold[2] % U64((1 << 30) - 10 ** 9), None)   # ids no batch brought
    E = bench_engine(args, 20_000_000)
    run = Run(E, bench.hyper(args))
    dev = [idr.on_device(b) for b in batches + [cold]]
    assert lf.above_l2_bound(batches)
    for j in (0, 1):
        run.step(batches[j], "train_dev", push=True, dev=dev[j])
    for j in (0, 1):
        run.step(batches[j], "train_dev", push=False, dev=dev[j])
    assert E.table_stats()["n_vrows"] == E.table_stats()["n_keys"]        # as bench.py requires after its warm-up
    run.step(batches[1], "val")
    run.step(batches[0], "predict")
    R = run.step(cold, "train_dev", push=False, dev=dev[2])
    assert E.table_stats()["n_vrows"] < E.table_stats()["n_keys"]
    assert R.n_amb <= R.amb_cap
    lf.assert_ran_without_lookup(E, batches[1])
    print(f"peak device memory {peak_gb():.1f} GB")


@pytest.mark.parametrize("V_dim", [0, 1, 10, 16, 40, 100, 128])
@pytest.mark.parametrize("valued", [False, True])
def test_widths_above_the_l2_bound(V_dim, valued):
    """lookup_free_step.big_batch: rows of 30..70 ids, three of 200..300 (long_row_nnz = 200), a hot id in 400 rows
    (hot_split = 64)"""
    rng = np.random.default_rng(500 + V_dim + valued)
    pool = np.unique(rng.integers(0, 1 << 40, 700000).astype(U64) * lf.GOLDEN)
    batches = [lf.big_batch(rng, pool[:400000], 70000, valued, pool[3]),
               lf.big_batch(rng, pool[200000:], 70000, valued, pool[3])]
    assert lf.above_l2_bound(batches)
    hp = dict(V_dim=V_dim, **lf.KW)
    # at V_dim >= 100 the worst-case forward bound leaves up to ~6e-3 of a warm step's keys within their bound of l1
    run = Run(capi.Engine(table_capacity=1 << 20, **lf.ENGINE, **hp), hp, hot_chunk=lf.ENGINE["hot_split"],
              amb_frac=F.AMB_FRAC if V_dim < 100 else 1e-2)
    dev = [idr.on_device(b) for b in batches]
    run.step(batches[0], "train_dev", push=True, dev=dev[0])
    run.step(batches[1], "train_dev", push=False, dev=dev[1])
    run.step(batches[0], "train_pred", push=False)


@pytest.mark.parametrize("vdim,hyper", [(64, "criteo_conf"), (10, "criteo_conf"), (64, "allV"), (32, "ftrl_l1")])
def test_criteo39_full_size(vdim, hyper):
    """Zipf hot keys in tens of thousands of rows (many k_hot_reduce chunks), the l1 threshold, sparse V rows"""
    args = bench_args(workload="criteo39", vdim=vdim, hyper=hyper)
    batches = [bench.gen_raw_batch(args, s) for s in (1, 2)]
    run = Run(bench_engine(args, 6_000_000), bench.hyper(args))
    dev = [idr.on_device(b) for b in batches]
    for j in (0, 1):
        run.step(batches[j], "train_dev", push=True, dev=dev[j])
    for j in (0, 1):
        run.step(batches[j], "train_dev", push=False, dev=dev[j])
    st = run.E.table_stats()
    assert hyper == "allV" or 0 < st["n_vrows"] < st["n_keys"]


def test_gisette_full_size():
    """1024 x 5000 valued, V_dim 64: k_fm_long, and every key in every row (pre-reduced in chunks)"""
    args = bench_args(workload="gisette", batch=1024, vdim=64)
    batches = [bench.gen_raw_batch(args, s) for s in (1, 2)]
    # l1 = 0 and rows of 5000: the worst-case forward bound is wide, and keys whose 1024 gradient terms nearly cancel
    # are ambiguous (up to ~8e-3 of the 5000)
    run = Run(bench_engine(args, 1 << 16), bench.hyper(args), amb_frac=1e-2)
    dev = [idr.on_device(b) for b in batches]
    run.step(batches[0], "train_dev", push=True, dev=dev[0])
    run.step(batches[1], "train_dev", push=False, dev=dev[1])
    run.step(batches[0], "train_pred", push=False)


def test_rcv1_full_size():
    args = bench_args(workload="rcv1", vdim=16, hyper="rcv1_conf")
    batches = [bench.gen_raw_batch(args, s) for s in (1, 2)]
    run = Run(bench_engine(args, 1 << 17), bench.hyper(args))
    dev = [idr.on_device(b) for b in batches]
    for j in (0, 1, 0):
        run.step(batches[j], "train_dev", push=j == 0, dev=dev[j])


@pytest.mark.parametrize("K", [8, 64])
@pytest.mark.parametrize("above", [False, True])
def test_both_sides_of_the_l2_plan_threshold(K, above):
    rng = np.random.default_rng(K + above)
    nnz = l2p.plan_threshold_nnz(K) + above
    pool = np.unique(rng.integers(0, 1 << 40, nnz // 16, dtype=U64))
    batches = [l2p.plan_batch(rng, nnz, pool, j == 1, pool[0]) for j in range(2)]
    assert all(l2p.plan_on(int(b[0][-1]), K) == above for b in batches)
    hp = dict(V_dim=K, **l2p.KW)
    run = Run(capi.Engine(table_capacity=1 << 20, **hp), hp)
    dev = [idr.on_device(b) for b in batches]
    run.step(batches[0], "train_dev", push=True, dev=dev[0])
    run.step(batches[1], "train_dev", push=False, dev=dev[1])
    run.step(batches[0], "train_dev", push=False, dev=dev[0])


def test_every_mutant_rejects_the_engine_step():
    """mid-size steps that exercise each deliberately wrong variant: a fresh step (InitV by the update), a warm valued
    step with a hot id in 400 rows and l2 > 0, and a step whose rows predict beyond +-20"""
    rng = np.random.default_rng(8)
    pool = np.unique(rng.integers(0, 1 << 40, 300000).astype(U64) * lf.GOLDEN)
    hp = dict(V_dim=16, **dict(lf.KW, V_threshold=0))
    run = Run(capi.Engine(table_capacity=1 << 20, **lf.ENGINE, **hp), hp, hot_chunk=lf.ENGINE["hot_split"])
    b0, b1 = (lf.big_batch(rng, pool, 20000, True, pool[3]) for _ in range(2))
    run.step(b0, "train_pred", push=True, mutants=("adagrad_on_new_initv",))
    run.step(b1, "train_pred", push=False,
             mutants=[m for m in F.MUTANTS if m not in ("adagrad_on_new_initv", "no_clamp")])
    hp = dict(V_dim=64, **dict(lf.KW, V_threshold=0, V_init_scale=4.0, l1=0.0))
    run = Run(capi.Engine(table_capacity=1 << 18, **hp), hp, amb_frac=3e-2)     # V rows of scale 4: loose forward bounds
    lens = rng.integers(20, 31, 5000)
    mk = lambda: idr.csr(rng, lens, pool[rng.integers(0, 20000, int(lens.sum()))], False)   # noqa: E731
    run.step(mk(), "train_pred", push=True)
    R = run.step(mk(), "train_pred", push=False, mutants=("no_clamp",))
    assert R.ok()
