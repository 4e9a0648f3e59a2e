"""The float64 one-step reference (fp64_step.py) grounded on the oracle, which is bit-identical to the compiled
reference: about 200 small random steps -- V_dim 0, 3, 8, 10, 64, 128, binary and valued, with and without the count
push, validation steps, hot keys, keys near the l1 threshold, V_threshold gating, lr_beta / V_lr_beta other than 1 --
leave the oracle's fp32 state, loss and penalty within the reference's bounds, and its InitV values, V-row pattern, table
size and rand_r state exactly as the reference says.  Then the sharpness check: every deliberately wrong variant of the
reference that applies at this size rejects the oracle's step that the true reference accepts."""
import numpy as np
import pytest

import fp64_step as F
from oracle import oracle as O
from util import oracle_state

U64 = np.uint64
GOLDEN = U64(0x9E3779B97F4A7C15)


def rand_batch(rng, pool, B, valued, hot=None, hot_rows=0, lens=(0, 21)):
    n = rng.integers(lens[0], lens[1], B)
    rows = [pool[rng.integers(0, len(pool), c)] for c in n]
    if hot is not None:
        for r in rng.choice(B, hot_rows, replace=False):
            rows[r] = np.concatenate([rows[r], np.array([hot], U64)])
    ids = np.concatenate(rows).astype(U64) if rows else np.zeros(0, U64)
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(U64)
    val = (rng.random(len(ids)).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, lab, ids, val


def oracle_step(M, hp, b, push, mode, **kw):
    """one step of the oracle: (reference factory, pre, post, observed); the factory takes a mutant"""
    o, l, i, v = b
    keys = F.batch_keys(i)[0]
    pre = oracle_state(M, keys)
    seed0, size0 = M.seed(), M.size()
    pr = M.sgd_step(o, i, v, l, is_train=mode == "train", push_cnt=push)
    post = oracle_state(M, keys)
    obs = dict(loss=float(pr[0]), penalty=float(pr[1]), nrows=float(pr[4]), n_keys_delta=M.size() - size0,
               rng_after=M.seed())

    def ref(mutant=None):
        return F.Reference(b, hp, pre, seed0, push, mode, "cpu", mutant=mutant, **kw)
    return ref, pre, post, obs


def hyper(V_dim, j):
    return dict(V_dim=V_dim, l1=(0.05, 0.3)[j % 2], l2=(0.01, 0.1)[j % 2], lr=(0.2, 0.5)[j % 2],
                lr_beta=(0.5, 2.0)[j % 2], V_lr=0.05, V_lr_beta=(0.3, 1.5)[j % 2], V_l2=0.02, V_init_scale=0.2,
                V_threshold=(2, 5)[j % 2], seed=11 + j)


@pytest.mark.parametrize("V_dim", [0, 3, 8, 10, 64, 128])
@pytest.mark.parametrize("valued", [False, True])
def test_oracle_steps_within_fp64_bounds(V_dim, valued):
    rng = np.random.default_rng(7 * V_dim + valued)
    hp = hyper(V_dim, V_dim + valued)
    M = O.Oracle(**hp)
    pool = np.unique(rng.integers(0, 1 << 40, 400).astype(U64) * GOLDEN)
    plan = [("train", True), ("train", False), ("train", True), ("val", False), ("train", False), ("train", True),
            ("train", False), ("val", False), ("train", True), ("train", False), ("train", False), ("train", True),
            ("val", False), ("train", False), ("train", True), ("train", False)]
    worst, amb, rows = 0.0, 0, 0
    for t, (mode, push) in enumerate(plan):
        sub = pool[: 150 + 16 * t]                             # new keys in every step
        b = rand_batch(rng, sub, 60, valued and t % 4 != 1, hot=pool[3], hot_rows=30)
        ref, pre, post, obs = oracle_step(M, hp, b, push, mode)
        R = F.check(ref(), pre, post, obs, what=f"V_dim {V_dim} valued {valued} step {t} {mode} push {push}")
        R.assert_ok()
        worst, amb = max(worst, R.max_ratio), amb + R.n_amb
        if mode == "train" and V_dim:
            rows += int((post[1] == 1).sum())
    assert worst > 0 and amb <= 2
    assert V_dim == 0 or rows > 0                               # V rows were made and updated


def mutant_case(name):
    """the oracle's step, and the reference, of a case the mutant applies to"""
    rng = np.random.default_rng(5)
    pool = np.unique(rng.integers(0, 1 << 40, 600).astype(U64) * GOLDEN)
    if name == "adagrad_on_new_initv":          # a fresh model's first step: every row InitV'd by the update
        hp = dict(hyper(8, 0), V_threshold=0, l1=0.0)
        M = O.Oracle(**hp)
        return oracle_step(M, hp, rand_batch(rng, pool, 200, False), True, "train")
    if name == "no_clamp":                      # V rows large enough that predictions pass +-20
        hp = dict(hyper(64, 0), V_threshold=0, l1=0.0, V_init_scale=4.0)
        M = O.Oracle(**hp)
        M.sgd_step(*[rand_batch(rng, pool[:200], 200, False, lens=(20, 31))[j] for j in (0, 2, 3, 1)], push_cnt=True)
        return oracle_step(M, hp, rand_batch(rng, pool[:200], 200, False, lens=(20, 31)), False, "train")
    hp = dict(hyper(8, 1), V_threshold=0)
    M = O.Oracle(**hp)
    valued = name == "xxp_uses_x"
    for _ in range(2):
        o, l, i, v = rand_batch(rng, pool, 500, valued, hot=pool[9], hot_rows=400)
        M.sgd_step(o, i, v, l, push_cnt=True)
    return oracle_step(M, hp, rand_batch(rng, pool, 500, valued, hot=pool[9], hot_rows=400), False, "train",
                       hot_chunk=64)


@pytest.mark.parametrize("mutant", F.MUTANTS)
def test_every_mutant_rejects_the_oracle(mutant):
    ref, pre, post, obs = mutant_case(mutant)
    F.check(ref(), pre, post, obs, what="true reference").assert_ok()
    R = F.check(ref(mutant), pre, post, obs, what=mutant)
    assert not R.ok(), f"{mutant} accepted: {R.summary()}"


# ---------------------------------------------------------------------------------------------------------------------
# k_fm_generic's summation order, emulated in float32
# ---------------------------------------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """fp32 fused multiply-add: a b of two fp32 values is exact in float64, so a b + c is rounded twice (float64,
    then fp32).  The first rounding adds at most 2^-53 relative, within the 2^-50 that fp64_step.U allows beyond 2^-24"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def warp_sum(v):
    """warp_sum (kernels_fm.cu:43-47) over the last axis (32 lanes): v += shfl_xor(v, o), o = 16 .. 1"""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lane ^ o]).astype(np.float32)
    return v[..., 0]


def emulate_generic_forward(off, x, w, V):
    """the prediction k_fm_generic (kernels_fm.cu:469-515) computes for each row, in its order and fp32 roundings:
    x, w per nonzero (float32 [nnz]), V[nnz, k] the nonzero's V row (zeros for a key without one, which the kernel skips:
    adding 0 is exact either way)"""
    B, k = len(off) - 1, V.shape[1]
    c = -(-k // 32)
    lens = np.diff(off.astype(np.int64))
    nmax = int(lens.max())
    chunks = -(-nmax // 32)
    X = np.zeros((B, chunks * 32), np.float32)
    W = np.zeros_like(X)
    Vt = np.zeros((B, nmax, c * 32), np.float32)
    for r in range(B):
        a, b = int(off[r]), int(off[r + 1])
        X[r, :b - a], W[r, :b - a] = x[a:b], w[a:b]
        Vt[r, :b - a, :k] = V[a:b]
    wsum = np.zeros((B, 32), np.float32)
    for ch in range(chunks):                                     # lane l: nonzeros l, l + 32, ... (:473-489)
        wsum = fmaf(X[:, ch * 32:(ch + 1) * 32], W[:, ch * 32:(ch + 1) * 32], wsum)
    A = (X[:, :nmax, None] * Vt).astype(np.float32)             # a = x_t V_f (:498)
    xv = np.zeros((B, c * 32), np.float32)
    acc2 = np.zeros((B, 32), np.float32)
    A4 = A.reshape(B, nmax, c, 32)
    for t in range(nmax):
        xv = (xv + A[:, t]).astype(np.float32)                  # xv[l] += a (:499)
        for j in range(c):
            acc2 = fmaf(A4[:, t, j], A4[:, t, j], acc2)          # acc2 = fmaf(a, a, acc2) (:500)
    pred = warp_sum(wsum)                                        # pred = 0 + wsum (:505-507)
    s1 = np.zeros((B, 32), np.float32)
    xv4 = xv.reshape(B, c, 32)
    for j in range(c):
        s1 = fmaf(xv4[:, j], xv4[:, j], s1)                      # (:510)
    d = (warp_sum(s1) - warp_sum(acc2)).astype(np.float32)
    pred = (pred + np.float32(0.5) * d).astype(np.float32)     # (:513)
    return np.clip(pred, np.float32(-20), np.float32(20))       # (:514)


@pytest.mark.parametrize("V_dim", [129, 256, 3073, 10000])
@pytest.mark.parametrize("valued", [False, True])
def test_generic_order_emulation_within_generic_bound(V_dim, valued):
    """random rows of up to 300 nonzeros, V rows of two scales (rows that stay inside +-20 and rows clamped), some keys
    without a V row, some x = 0 and negative x"""
    rng = np.random.default_rng(V_dim + valued)
    lens = np.array([0, 1, 3, 17, 40, 100, 300, 300] + ([] if V_dim > 3072 else list(rng.integers(0, 300, 8))))
    pool = np.unique(rng.integers(0, 1 << 40, 1200).astype(U64) * GOLDEN)
    o, l, ids, v = csr(rng,lens, pool[rng.integers(0, len(pool), int(lens.sum()))], valued)
    if valued:
        v[rng.random(len(v)) < 0.05] = 0
    keys, lidx, _ = F.batch_keys(ids)
    Uk = len(keys)
    scal = np.zeros((Uk, 4), np.float32)
    scal[:, 1] = rng.normal(0, 0.3, Uk).astype(np.float32)
    hasv = np.where(rng.random(Uk) < 0.9, 1, 0).astype(np.int32)
    scale = np.where(rng.random(Uk) < 0.5, 0.02, 0.3)[:, None]
    V = (rng.uniform(-1, 1, (Uk, V_dim)) * scale).astype(np.float32) * (hasv == 1)[:, None]
    pre = (scal, hasv, V, np.zeros_like(V))
    x = v if valued else np.ones(len(ids), np.float32)
    emu = emulate_generic_forward(o, x, scal[lidx, 1], V[lidx])
    ref = F.Reference((o, l, ids, v), dict(V_dim=V_dim), pre, 0, mode="predict", order="generic")
    err = np.abs(emu.astype(np.float64) - ref.pred.numpy())
    e = ref.e_pred.numpy()
    assert (err <= e).all(), f"rows {np.nonzero(err > e)[0]}: error {err.max():.3g}, bound {e[np.argmax(err / e)]:.3g}"
    assert (np.abs(ref.pred.numpy()) == 20).any() and (np.abs(ref.pred.numpy()) < 20).any()   # both kinds of rows
    print(f"V_dim {V_dim} valued {valued}: max error / bound {float((err / np.where(e > 0, e, 1)).max()):.3g}")


def csr(rng, lens, ids, valued):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(U64)
    val = (rng.random(len(ids)).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(len(lens)) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, lab, ids, val


# ---------------------------------------------------------------------------------------------------------------------
# validation steps on ids the table never saw
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("val_inserts", [True, False])
def test_validation_on_unseen_ids(val_inserts):
    """the reference inserts a validation batch's absent keys (its Pull); the fused steps do not.  The oracle's step is
    the first; the second is the same step with the state left as it was.  Each is accepted by the reference with the
    matching val_inserts and rejected by the other"""
    rng = np.random.default_rng(41)
    hp = hyper(8, 0)
    M = O.Oracle(**hp)
    pool = np.unique(rng.integers(0, 1 << 40, 600).astype(U64) * GOLDEN)
    for _ in range(2):
        o, l, i, v = rand_batch(rng, pool[:300], 80, False)
        M.sgd_step(o, i, v, l, push_cnt=True)
    b = rand_batch(rng, pool, 80, True)                     # half of the ids unseen
    ref, pre, post, obs = oracle_step(M, hp, b, False, "val")
    assert (pre[1] < 0).sum() > 20 and obs["n_keys_delta"] == (pre[1] < 0).sum()
    if not val_inserts:
        post, obs = pre, dict(obs, n_keys_delta=0)
    F.check(F.Reference(b, hp, pre, M.seed(), False, "val", val_inserts=val_inserts), pre, post, obs).assert_ok()
    R = F.check(F.Reference(b, hp, pre, M.seed(), False, "val", val_inserts=not val_inserts), pre, post, obs)
    assert not R.ok(), R.summary()


# ---------------------------------------------------------------------------------------------------------------------
# one InitV stream per owner: one worker's step over S oracle owners (shard_sim)
# ---------------------------------------------------------------------------------------------------------------------
def owner_steps(S, steps, hp, batch_fn):
    """every step of shard_sim.simulate with S owners: (batch, push, pre, post, streams, observed) for the batch of
    worker 0, whose keys are all the owners receive (the other workers' batches are empty).  The state of the batch's
    keys is the owners' merged in key order; each owner's rng state before the step seeds its own stream"""
    import shard_sim
    from difacto_b200.sharded import shard_bounds_np
    out = []
    for t in range(steps):
        before = shard_sim.simulate(S, t, hp, batch_fn)
        after = shard_sim.simulate(S, t + 1, hp, batch_fn)
        off, idx, val, lab = batch_fn(0, t)
        keys = F.batch_keys(idx)[0]
        bounds = shard_bounds_np(keys, S)

        def merged(shards):
            parts = [oracle_state(shards[s].M, keys[bounds[s]:bounds[s + 1]]) for s in range(S)]
            return tuple(np.concatenate([p[j] for p in parts]) for j in range(4))
        seeds = [sh.M.seed() for sh in before[0]]
        prog = after[2][t][0]
        obs = dict(loss=float(prog[0]), penalty=float(prog[1]), rng_after=[sh.M.seed() for sh in after[0]],
                   n_keys_delta=sum(a.M.size() - b.M.size() for a, b in zip(after[0], before[0])))
        out.append(((off, lab, idx, val), t < 2, merged(before[0]), merged(after[0]), (bounds, seeds), obs))
    return out


@pytest.mark.parametrize("S", [2, 3, 8])
def test_per_owner_initv_streams(S):
    """the simulated sharded store with one worker: every step within the reference's bounds when each owner draws its
    own stream, and rejected by the single-stream reference whenever two owners drew InitV rows"""
    import shard_sim
    hp = dict(hyper(8, S), V_threshold=1)
    empty = (np.zeros(5, U64), np.zeros(0, U64), None, np.ones(4, np.float32))

    def batch_fn(rank, step):
        if rank:
            return empty
        return shard_sim.raw_batch(0, step, step % 2 == 1, B=80, ids=300, hot=True, seed=S)
    rejected = 0
    for t, (b, push, pre, post, streams, obs) in enumerate(owner_steps(S, 4, hp, batch_fn)):
        ref = F.Reference(b, hp, pre, 0, push, "train", "cpu", streams=streams)
        R = F.check(ref, pre, post, obs, what=f"S {S} step {t}")
        R.assert_ok()
        bounds = streams[0]
        drew = [int(((post[1] == 1) & (pre[1] != 1))[bounds[s]:bounds[s + 1]].sum()) for s in range(S)]
        print(f"{R.summary()}; new rows per owner {drew}")
        if sum(d > 0 for d in drew) >= 2:
            R1 = F.check(F.Reference(b, hp, pre, streams[1][0], push, "train", "cpu"), pre, post,
                         dict(obs, rng_after=obs["rng_after"][0]), what="one stream")
            assert not R1.ok() and any("InitV" in f for f in R1.fail), R1.summary()
            rejected += 1
    assert rejected >= 2
