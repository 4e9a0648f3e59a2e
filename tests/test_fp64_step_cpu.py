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
