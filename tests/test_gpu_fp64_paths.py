"""The engine's other training paths against the float64 one-step reference (fp64_step.py), as test_gpu_fp64_step.py
holds the sorted raw-id step: every key a step touches within its bound, at least 100 k keys outside the batch
unchanged bit for bit, the AUC of the returned predictions against float64.

Paths: V_dim above 128 (k_fm_generic with its row of XV in dynamic shared memory, k_update_dense_generic, the localizer
that brings the key count to the host), from 129 to the engine's maximum of 10000, across the 48 KB shared-memory
opt-in at 3072 / 3073; scatter=atomic at every lane-group width (k_fm_fast<K, 1> + k_update_fast<K>) and at two
widths that take the generic kernels, through the raw and the host-localized step; force_generic and the atomic
scatter at the benchmark's shapes; the plugin calls in the reference's BatchPluginCalls order (dfb_push_feacnt,
dfb_pull, dfb_predict, dfb_evaluate, dfb_auc, dfb_calc_grad, dfb_push_grad: the ragged layout, k_grad_finalize,
k_update_ragged).
Validation steps on unseen ids: the fused steps insert nothing, the plugin calls insert every key (as the reference's
Pull does).  Then the sharpness check on one generic, one atomic and one plugin step, and no_clamp on validation and
predict steps whose rows pass +-20 on each path.  Each case prints its largest error-to-bound ratio and its count of
ambiguous keys."""
import time

import numpy as np
import pytest

import bench
import fp64_step as F
import test_gpu_fp64_step as S
import test_gpu_id_range as idr
import test_gpu_lookup_free_step as lf
from oracle import oracle as O

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

U64 = np.uint64
EXACT = (8, 16, 32, 64, 128)          # the lane-group widths: the atomic scatter's specialised kernels
SHARP = ("drop_hot_occ", "xxp_uses_x", "post_update_V_in_xxp", "swap_tile_neighbour", "no_l2_in_grad_w")


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class PathRun(S.Run):
    """Run for the paths other than the sorted step: the forward order and the penalty launch of each kind of step,
    fused validation steps that insert nothing, the host-localized step and the plugin calls.

    scatter / force_generic as the engine was created; plugin: the steps are the plugin calls (whose dfb_predict and
    dfb_calc_grad always run k_fm_generic, engine.cu:1065, :1105)"""

    def __init__(self, E, hp, scatter="sorted", force_generic=False, plugin=False, amb_frac=F.AMB_FRAC, hot_chunk=256):
        super().__init__(E, hp, hot_chunk=hot_chunk, amb_frac=amb_frac)
        k = hp["V_dim"]
        fast = 0 <= k <= 128 and not force_generic                  # fm_fast_supported (dfb_internal.cuh:201)
        assert plugin or not (fast and scatter == "sorted"), "the sorted training step is test_gpu_fp64_step.py's"
        # training: launch_fm sends the atomic scatter to k_fm_fast<K, 1> at the exact widths (kernels_fm.cu:690-693)
        self.order = {"train": "sorted" if fast and k in EXACT else "generic",
                      "val": "sorted" if fast else "generic", "predict": "sorted" if fast else "generic"}
        sms = num_sms()
        # launch_update_dense (kernels_table.cu:1273-1289): k_update_fast<K> at the exact widths, whatever the forward
        self.pen = {"train": F.pen_partial_update_fast(sms) if k in EXACT else F.pen_partial_warp_per_key(sms),
                    "val": F.pen_partial_warp_per_key(sms)}      # k_penalty (engine.cu:385-386)

    def hold(self, b, mode, push, pre, post, seed0, obs, order, pen, val_inserts, what, mutants=(), t_step=0.0,
             streams=None):
        ref = F.Reference(b, self.hp, pre, seed0, push, mode, "cuda", hot_chunk=self.hot_chunk, order=order,
                          val_inserts=val_inserts, streams=streams)
        t0 = time.perf_counter()
        R = F.check(ref, pre, post, obs, what=what, pen_partial=pen, amb_frac=self.amb_frac)
        print(f"{R.summary()}; engine {t_step:.2f} s, reference + comparison {time.perf_counter() - t0:.1f} s, "
              f"keys {ref.U}")
        R.assert_ok()
        self.last_n_push = ref.n_push
        del ref
        for m in mutants:
            Rm = F.check(F.Reference(b, self.hp, pre, seed0, push, mode, "cuda", mutant=m, hot_chunk=self.hot_chunk,
                                     order=order, val_inserts=val_inserts, streams=streams), pre, post, obs, what=m,
                         pen_partial=pen)
            assert not Rm.ok(), f"the {m} variant of the reference accepts the engine's step ({what}): {Rm.summary()}"
            print(f"  {m} rejects it: {Rm.fail[0] if Rm.fail else Rm.summary()}")
        self.reports.append(R)
        torch.cuda.empty_cache()
        return R

    def remember(self, keys, cnt):
        allk = np.concatenate([self.seen, keys])
        allc = np.concatenate([self.seen_cnt, cnt])
        self.seen, inv = np.unique(allk, return_inverse=True)
        self.seen_cnt = np.zeros(len(self.seen), np.int64)
        np.add.at(self.seen_cnt, inv, allc)

    def step(self, b, kind, push=False, mutants=()):
        """kind: raw (train_step_raw), host (train_step on the batch localized on the host), val, predict, plugin
        (a training step of plugin calls) or plugin_val (pull, predict, evaluate, auc)"""
        E, k = self.E, self.hp["V_dim"]
        o, l, i, v = b
        keys, lidx, cnt = F.batch_keys(i)
        pre = E.read_entries(keys)
        out = self.outside(keys)
        out_pre = E.read_entries(out)
        seed0, st0 = E.rng_state(), E.table_stats()
        t0 = time.perf_counter()
        plugin = kind.startswith("plugin")
        if plugin:
            obs = self._plugin(b, keys, lidx, cnt, push, kind == "plugin", pre, seed0)
        else:
            if kind == "raw":
                pr, pred = E.train_step_raw(o, i, v, l, push_cnt=push, is_train=True, want_pred=True)
            elif kind == "host":
                pr, pred = E.train_step(o, lidx.astype(np.uint32), v, l, keys, cnt.astype(np.float32) if push else None,
                                        is_train=True, want_pred=True)
            elif kind == "val":
                pr, pred = E.train_step_raw(o, i, v, l, push_cnt=False, is_train=False, want_pred=True)
            else:
                pr, pred = E.predict_raw(o, i, v, l)
            obs = dict(loss=pr.loss, penalty=pr.penalty, nrows=pr.nrows, new_keys=pr.new_keys, new_vrows=pr.new_vrows,
                       pred=pred, auc=pr.auc, label=l)
        t_step = time.perf_counter() - t0
        post = E.read_entries(keys)
        st1 = E.table_stats()
        obs.update(n_keys_delta=st1["n_keys"] - st0["n_keys"], n_vrows_delta=st1["n_vrows"] - st0["n_vrows"],
                   rng_after=E.rng_state())
        mode = {"raw": "train", "host": "train", "plugin": "train", "plugin_val": "val"}.get(kind, kind)
        if mode != "train" and not plugin:
            assert st1["n_keys"] == st0["n_keys"], f"a fused {kind} step grew the table"
        R = self.hold(b, mode, push, pre, post, seed0, obs, "generic" if plugin else self.order[mode],
                      None if plugin else self.pen.get(mode), plugin, f"{kind} push={push}", mutants, t_step)
        F.assert_unchanged(out_pre, E.read_entries(out), out, f"{kind} push={push}")
        if mode == "train" or plugin:
            self.remember(keys, cnt)
        self.last_obs = obs
        return R

    def _plugin(self, b, keys, lidx, cnt, push, train, pre, seed0):
        """SGDLearner::BatchPluginCalls (sgd_learner.cc:547-573): the Pull returns exactly the pre-step rows (with the
        count push's InitV rows), then predict / evaluate / auc, and for a training step calc_grad and push_grad.  The
        penalty is the learner's, on the host: not an engine output"""
        E, k = self.E, self.hp["V_dim"]
        o, l, i, v = b
        if push:
            E.push_feacnt(keys, cnt.astype(np.float32))
        vals, lens = E.pull(keys)
        # what the Pull must return: the reference's pulled w and V rows, bit for bit
        ref = F.Reference(b, self.hp, pre, seed0, push, "train" if train else "val", "cuda")
        want_lens = np.where(ref.hv_pull, k + 1, 1).astype(np.int32) if k else np.zeros(0, np.int32)
        assert np.array_equal(lens, want_lens), "pulled lens differ from the reference's V-row pattern"
        if k:
            w_pos, V_pos = O.get_pos(lens)
            hv = np.nonzero(ref.hv_pull)[0]
            got_V = vals[V_pos[hv][:, None] + np.arange(k)]
            assert np.array_equal(got_V, ref.Vp.cpu().numpy()[hv]), "pulled V rows differ (count-push InitV rows?)"
        else:
            w_pos = V_pos = None
        got_w = vals[w_pos] if k else vals
        assert np.array_equal(got_w, pre[0][:, 1]), "pulled w differ from the pre-step state"
        del ref
        pred = E.predict(o, lidx.astype(np.uint32), v, vals, w_pos, V_pos)
        loss, auc = E.evaluate(l, pred), E.auc(l, pred)
        if train:
            grad = E.calc_grad(o, lidx.astype(np.uint32), v, l, vals, pred, w_pos, V_pos)
            E.push_grad(keys, grad, lens if k else None)
        return dict(loss=loss, pred=pred, auc=auc, label=l)


def mid_batch(rng, pool, B, valued, hot, long_rows=(200, 301)):
    """rows of 0..40 ids, three of long_rows ids, `hot` in 400 rows; valued: x in [-.5, 1.5), 5 % of them 0"""
    lens = rng.integers(0, 41, B)
    lens[rng.choice(B, 3, replace=False)] = rng.integers(*long_rows, 3)
    ids = pool[rng.integers(0, len(pool), int(lens.sum()))]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    has = np.nonzero(lens > 0)[0]
    ids[starts[rng.choice(has, 400, replace=False)]] = hot
    b = idr.csr(rng, lens, ids, valued)
    if valued:
        b[3][rng.random(len(ids)) < 0.05] = 0
    return b


def pool_of(rng, n):
    return np.unique(rng.integers(0, 1 << 40, n).astype(U64) * lf.GOLDEN)


# ---------------------------------------------------------------------------------------------------------------------
# V_dim > 128: the generic kernels
# ---------------------------------------------------------------------------------------------------------------------
# V_init_scale by width: the rows' Q = sum x^2 V_f^2 enters k_fm_generic's bound with gamma(n ceil(k / 32) + 7), so the
# widest rows keep their V small enough that the forward bound stays far below the gradients' size
WIDE = [(129, False), (129, True), (130, False), (131, True), (132, False), (160, True), (255, False), (256, False),
        (256, True), (257, True), (1000, False), (3072, True), (3073, False), (10000, False)]


def wide_hp(V_dim):
    return dict(V_dim=V_dim, **dict(lf.KW, V_init_scale=0.01 if V_dim <= 1000 else 0.005 if V_dim < 10000 else 0.001))


@pytest.mark.parametrize("V_dim,valued", WIDE)
def test_generic_widths(V_dim, valued):
    """two training steps with the count push (the second gives InitV rows to keys the first made nonzero), one
    without, a validation step on a batch with unseen ids (nothing inserted), a predict step.  129 .. 132: the row
    stride rounded up to 132 and a partial last float4; 255 .. 257: the lane loop l += 32;
    3072 / 3073: either side of the 48 KB shared-memory opt-in (kernels_fm.cu:708-709); 10000: the maximum, few keys"""
    rng = np.random.default_rng(1000 + V_dim + valued)
    small = V_dim == 10000
    pool = pool_of(rng, 3000 if small else 30000)
    B = 500 if small else 2000
    b0 = mid_batch(rng, pool[:len(pool) * 2 // 3], B, valued, pool[5])
    b1 = mid_batch(rng, pool[len(pool) // 3:], B, valued, pool[5])
    unseen = np.concatenate([pool, pool_of(rng, len(pool) // 2) + U64(1)])
    b2 = mid_batch(rng, unseen, B, valued, pool[7])
    hp = wide_hp(V_dim)
    cap = 1 << 14 if small else 1 << 17
    run = PathRun(capi.Engine(table_capacity=cap, V_capacity=cap, **lf.ENGINE, **hp), hp,
                  hot_chunk=lf.ENGINE["hot_split"])
    run.step(b0, "raw", push=True)
    run.step(b1, "raw", push=True)
    assert run.last_n_push > 0                                                  # the count push's InitV rows
    run.step(b0, "raw")
    assert len(np.setdiff1d(F.batch_keys(b2[2])[0], run.seen)) > 100          # ids the table never saw
    run.step(b2, "val")                                                         # (asserts n_keys did not change)
    run.step(b0, "predict")
    print(f"peak device memory {S.peak_gb():.1f} GB")


def test_generic_pipelined_steps_in_flight():
    """two raw steps in flight through train_step_raw_async and prefetch_raw at V_dim 257: the localizer of this path
    brings each batch's key count to the host while the previous step runs.  The batches' keys are disjoint, so each
    step's pre-step state is read before both; the second step's rng state is the first's seed jumped by its new rows"""
    rng = np.random.default_rng(257)
    pool = pool_of(rng, 40000)
    hp = wide_hp(257)
    E = capi.Engine(table_capacity=1 << 17, **lf.ENGINE, **hp)
    run = PathRun(E, hp, hot_chunk=lf.ENGINE["hot_split"])
    run.step(mid_batch(rng, pool[:20000], 2000, True, pool[5]), "raw", push=True)
    bs = [mid_batch(rng, pool[:20000], 2000, True, pool[5]), mid_batch(rng, pool[20000:], 2000, False, pool[20005])]
    ks = [F.batch_keys(b[2]) for b in bs]
    assert len(np.intersect1d(ks[0][0], ks[1][0])) == 0
    pres = [E.read_entries(kc[0]) for kc in ks]
    out = run.outside(np.union1d(ks[0][0], ks[1][0]))
    out_pre = E.read_entries(out)
    seed0, st0 = E.rng_state(), E.table_stats()
    o, l, i, v = bs[0]
    E.train_step_raw_async(len(l), o, i, v, l, push_cnt=True)
    o1, l1, i1, v1 = bs[1]
    E.prefetch_raw(len(l1), o1, i1, v1, l1)
    E.train_step_raw_async(len(l1), o1, i1, v1, l1, push_cnt=False)
    prs = [E.wait_step(), E.wait_step()]
    st1 = E.table_stats()
    assert st1["n_keys"] - st0["n_keys"] == sum(int((p[1] < 0).sum()) for p in pres)
    seed = seed0
    for j, (b, (keys, _, cnt), pre, pr) in enumerate(zip(bs, ks, pres, prs)):
        obs = dict(loss=pr.loss, penalty=pr.penalty, nrows=pr.nrows, new_keys=pr.new_keys, new_vrows=pr.new_vrows)
        if j == 1:
            obs["rng_after"] = E.rng_state()
        run.hold(b, "train", j == 0, pre, E.read_entries(keys), seed, obs, "generic", run.pen["train"], False,
                 f"in flight, step {j}")
        seed = int(F.lcg_jump(seed, 3 * 257 * pr.new_vrows)[0])
        run.remember(keys, cnt)
    F.assert_unchanged(out_pre, E.read_entries(out), out, "two steps in flight")


def test_generic_batch_outside_id_bits_changes_nothing():
    """id_bits = 30 at V_dim 130: a batch with one id at 2^32 (above the sorted range) is dropped -- the step fails
    with the id range error, and
    every key of it, and of the batches before, is what it was"""
    rng = np.random.default_rng(30)
    pool = np.unique(idr.rand_u64(rng, 20000, 30))        # (id_bits = 30 sorts the ids below 2^32)
    hp = wide_hp(130)
    E = capi.Engine(table_capacity=1 << 16, id_bits=30, **lf.ENGINE, **hp)
    run = PathRun(E, hp, hot_chunk=lf.ENGINE["hot_split"])
    good = [mid_batch(rng, pool, 1000, j == 1, pool[3]) for j in range(2)]
    run.step(good[0], "raw", push=True)
    run.step(good[1], "raw")
    o, l, i, v = mid_batch(rng, pool, 1000, False, pool[3])
    bad = idr.csr(rng, np.diff(o.astype(np.int64)) + np.eye(len(l), dtype=np.int64)[-1],
                  np.concatenate([i, np.array([1 << 32], U64)]), False)
    keys = np.union1d(F.batch_keys(bad[2])[0], run.seen)
    before, seed0, st0 = E.read_entries(keys), E.rng_state(), E.table_stats()
    with pytest.raises(capi.DfbError, match="id_bits = 30"):
        E.train_step_raw(*[bad[j] for j in (0, 2, 3, 1)], push_cnt=False, is_train=True)
    F.assert_unchanged(before, E.read_entries(keys), keys, "dropped batch")
    assert E.rng_state() == seed0 and E.table_stats() == st0
    run.step(good[0], "raw")                                    # and the next step is held to the reference as usual


# ---------------------------------------------------------------------------------------------------------------------
# the benchmark's shapes on the non-sorted paths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [dict(scatter="atomic"), dict(force_generic=1)], ids=["atomic", "force_generic"])
def test_flagship_non_sorted(extra):
    """bench.py's flagship (65536 x 100, V_dim 64, allV): pass 0 with the count push, then pass 1, on one batch (its
    ~6.5 M keys in a table of 8 M: the GPU is shared)"""
    args = S.bench_args()
    b = bench.gen_raw_batch(args, 1)
    E = S.bench_engine(args, 8_000_000, **extra)
    run = PathRun(E, bench.hyper(args), scatter=extra.get("scatter", "sorted"), force_generic="force_generic" in extra)
    run.step(b, "raw", push=True)
    run.step(b, "raw")
    assert E.table_stats()["n_vrows"] == E.table_stats()["n_keys"]
    print(f"peak device memory {S.peak_gb():.1f} GB")
    E.close()


@pytest.mark.parametrize("args", [S.bench_args(vdim=256, batch=16384),
                                  S.bench_args(workload="criteo39", vdim=160, hyper="criteo_conf"),
                                  S.bench_args(workload="gisette", batch=256, vdim=160)],
                         ids=["synthetic_V256", "criteo39_V160", "gisette_V160"])
def test_wide_at_bench_shapes(args):
    """pass 0 with the count push, then pass 1, on one batch (tables sized to its keys: the GPU is shared)"""
    b = bench.gen_raw_batch(args, 1)
    cap = {"synthetic": 2_000_000, "criteo39": 2_000_000, "gisette": 1 << 14}[args.workload]
    gisette = args.workload == "gisette"
    # gisette: l1 = 0 and rows of 5000 -- keys whose 256 gradient terms nearly cancel are ambiguous, as at V_dim 64
    # (test_gpu_fp64_step.py's gisette case)
    run = PathRun(S.bench_engine(args, cap), bench.hyper(args), amb_frac=1e-2 if gisette else F.AMB_FRAC)
    run.step(b, "raw", push=True)
    run.step(b, "raw")
    print(f"peak device memory {S.peak_gb():.1f} GB")


# ---------------------------------------------------------------------------------------------------------------------
# scatter=atomic at every lane-group width, and at two that take the generic kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [8, 16, 32, 64, 128, 10, 40])
def test_atomic_scatter(V_dim):
    rng = np.random.default_rng(2000 + V_dim)
    pool = pool_of(rng, 30000)
    bs = [mid_batch(rng, pool[:20000], 2000, j % 2 == 1, pool[5]) for j in range(2)]
    hp = dict(V_dim=V_dim, **lf.KW)
    run = PathRun(capi.Engine(table_capacity=1 << 17, scatter="atomic", **lf.ENGINE, **hp), hp, scatter="atomic",
                  hot_chunk=lf.ENGINE["hot_split"])
    run.step(bs[0], "raw", push=True)
    run.step(bs[1], "host")
    run.step(bs[0], "host", push=True)
    run.step(bs[1], "raw")


# ---------------------------------------------------------------------------------------------------------------------
# the plugin calls
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [0, 10, 64, 129])
def test_plugin_calls(V_dim):
    """two steps with the count push -- the second gives InitV rows to keys the first made nonzero, and its Pull must
    return them -- one without, then a validation step (pull, predict, evaluate, auc) on a batch with unseen ids: the
    Pull inserts them"""
    rng = np.random.default_rng(3000 + V_dim)
    pool = pool_of(rng, 30000)
    hp = dict(V_dim=V_dim, **lf.KW)
    run = PathRun(capi.Engine(table_capacity=1 << 17, **lf.ENGINE, **hp), hp, plugin=True,
                  hot_chunk=lf.ENGINE["hot_split"])
    run.step(mid_batch(rng, pool[:20000], 2000, False, pool[5]), "plugin", push=True)
    run.step(mid_batch(rng, pool[10000:], 2000, True, pool[5]), "plugin", push=True)
    assert V_dim == 0 or run.last_n_push > 0                    # the count push's InitV rows, pulled bit for bit
    run.step(mid_batch(rng, pool[:20000], 2000, True, pool[5]), "plugin")
    b = mid_batch(rng, np.concatenate([pool, pool_of(rng, 10000) + U64(1)]), 2000, True, pool[7])
    new = len(np.setdiff1d(F.batch_keys(b[2])[0], run.seen))
    n0 = run.E.table_stats()["n_keys"]
    assert new > 100
    run.step(b, "plugin_val")
    assert run.E.table_stats()["n_keys"] - n0 == new


# ---------------------------------------------------------------------------------------------------------------------
# sharpness: every applicable wrong variant rejects the engine's step
# ---------------------------------------------------------------------------------------------------------------------
SHARP_PATHS = {"generic_V256": (256, dict(), "raw"), "atomic_V64": (64, dict(scatter="atomic"), "raw"),
               "plugin_V64": (64, dict(), "plugin")}


@pytest.mark.parametrize("path", list(SHARP_PATHS))
def test_every_mutant_rejects_the_engine_step(path):
    """a fresh step (InitV by the update) and a warm valued step with a hot id in 400 rows and l2 > 0.  (no_clamp:
    test_no_clamp_rejects_predictions_beyond_20)"""
    K, extra, kind = SHARP_PATHS[path]
    scatter = extra.get("scatter", "sorted")
    rng = np.random.default_rng(K + len(path))
    pool = pool_of(rng, 300000)
    # V rows of 0.05 at V_dim 256: the rows of 30..70 ids keep k_fm_generic's Q-chain bound small
    hp = dict(V_dim=K, **dict(lf.KW, V_threshold=0, V_init_scale=0.2 if K <= 64 else 0.05))
    run = PathRun(capi.Engine(table_capacity=1 << 20, **lf.ENGINE, **extra, **hp), hp, scatter=scatter,
                  plugin=kind == "plugin", hot_chunk=lf.ENGINE["hot_split"])
    b0, b1 = (lf.big_batch(rng, pool, 20000, True, pool[3]) for _ in range(2))
    run.step(b0, kind, push=True, mutants=("adagrad_on_new_initv",))
    run.step(b1, kind, mutants=SHARP)


NO_CLAMP_PATHS = {"generic_V256": (256, dict(), "raw", False),
                  "force_generic_V64": (64, dict(force_generic=1), "raw", True),
                  "atomic_V64": (64, dict(scatter="atomic"), "raw", False), "plugin_V64": (64, dict(), "plugin", False)}


@pytest.mark.parametrize("path", list(NO_CLAMP_PATHS))
def test_no_clamp_rejects_predictions_beyond_20(path):
    """V rows of scale ~4 (InitV by an unchecked training step) take most rows of 8..12 ids past +-20; a validation and
    a predict step (plugin: pull, dfb_predict, evaluate, auc) return them clamped, and the no_clamp variant of the
    reference rejects both.  (A training step on such rows leaves more keys within their bound of FTRL's branch than
    the cap allows: the held steps here have no FTRL branch)"""
    K, extra, kind, fg = NO_CLAMP_PATHS[path]
    rng = np.random.default_rng(20 + K + len(path))
    pool = pool_of(rng, 40000)
    hp = dict(V_dim=K, **dict(lf.KW, V_threshold=0, V_init_scale=4.0 * (64 / K) ** 0.25, l1=0.0))
    E = capi.Engine(table_capacity=1 << 17, **extra, **hp)
    run = PathRun(E, hp, scatter=extra.get("scatter", "sorted"), force_generic=fg, plugin=kind == "plugin")
    lens = rng.integers(8, 13, 5000)
    mk = lambda: idr.csr(rng, lens, pool[rng.integers(0, 20000, int(lens.sum()))], False)   # noqa: E731
    for _ in range(2):                                  # the rows' keys get their (large) InitV rows
        o, l, i, v = mk()
        E.train_step_raw(o, i, v, l, push_cnt=True, is_train=True)
        run.remember(*F.batch_keys(i)[::2])
    assert E.table_stats()["n_vrows"] > 10000
    for step in (("plugin_val",) if kind == "plugin" else ("val", "predict")):
        run.step(mk(), step, mutants=("no_clamp",))
        pred = run.last_obs["pred"]
        assert (np.abs(pred) == 20).mean() > 0.2 and (np.abs(pred) < 20).any(), "rows past +-20 and rows inside"
