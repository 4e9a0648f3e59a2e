"""Every V_dim from 0 to 128 on the specialised sorted kernels (single-GPU fused step and the NVLink-sharded store).

A V_dim that is not one of the lane-group widths K in {8,16,32,64,128} runs on the smallest K above it, with rows of
stride ks = V_dim rounded up to 4 and the lanes beyond ks idle.  Checked here against the oracle (tolerances of
test_gpu_parity.py: InitV stream, has-V pattern and feature counts exact), against the generic kernels
(force_generic=1, the path these widths took before) and against themselves (bit-reproducible):
  * trajectories at widths that cover every K, whole idle lanes and partial last float4s;
  * the pad columns [V_dim, ks) stay 0 with V_lr_beta = 0 (AdaGrad would divide by cg = 0 there);
  * a dropped raw batch (id outside id_bits) changes nothing;
  * the sharded store at V_dim 0, 10, 40 with 1..3 ranks on one GPU, and the C++ CLI on 2 GPUs;
  * V_dim 129 stays on the generic kernels, and the sharded store refuses it.
"""
import os
import subprocess
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import oracle as O  # noqa: E402
from shard_sim import STATE_TOL, all_keys, check_vs_simulation, raw_batch, run_local  # noqa: E402
from util import assert_close, localized, oracle_state, rand_batch  # noqa: E402
import test_gpu_id_range as idr  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(l1=0.3, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=4, V_l2=0.02, V_init_scale=0.2, seed=5)


def keys_of(batches):
    return np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b in batches]))


def run_traj(kw, batches, epochs, raw, val_every=4, **engine_kw):
    """the engine and the oracle over the same batches (localized or raw steps, every val_every-th a validation step);
    per-step loss / penalty / rows as test_gpu_parity.run_both"""
    M = O.Oracle(**kw)
    E = capi.Engine(table_capacity=1 << 16, **engine_kw, **kw)
    t = 0
    for ep in range(epochs):
        for (o, l, i, v) in batches:
            is_train = not (val_every and t % val_every == val_every - 1)
            push = ep == 0 and is_train
            ref = M.sgd_step(o, i, v, l, is_train, push)
            if raw:
                pr = E.train_step_raw(o, i, v, l, push_cnt=push, is_train=is_train)
            else:
                b = localized((o, l, i, v))
                pr = E.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"] if push else None, is_train)
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
    assert E.rng_state() == M.seed()
    return ohasv


# ---------------------------------------------------------------------------------------------------------------------
# 1. single-GPU trajectories: every K (8: 0..8, 16: 10, 12, 32: 20, 64: 40, 128: 100, 127), idle lanes, partial float4s
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("raw", [False, True], ids=["localized", "raw"])
@pytest.mark.parametrize("V_dim", [0, 1, 3, 4, 6, 10, 12, 20, 40, 100, 127])
def test_any_vdim_trajectory_vs_oracle(V_dim, raw):
    rng = np.random.default_rng(2000 + V_dim)
    kw = dict(V_dim=V_dim, **KW)
    batches = [rand_batch(rng, 128, 30, 400, j % 2 == 0) for j in range(5)]      # binary and valued
    M, E = run_traj(kw, batches, epochs=4, raw=raw)
    ohasv = compare_state(M, E, keys_of(batches))
    if V_dim:
        assert (ohasv == 1).sum() > 10


# ---------------------------------------------------------------------------------------------------------------------
# 2. bit-reproducible and on the sorted path, hot keys included; within rounding of the generic kernels
# ---------------------------------------------------------------------------------------------------------------------
def hot_batches(rng, n=4):
    """a key in every row (over hot_split = 256 occurrences: the chunked pre-reduction) and ~40-occurrence keys"""
    out = []
    for j in range(n):
        o, l, i, v = rand_batch(rng, 1000, 14, 300, j % 2 == 1, min_nnz=2)
        i[o[:-1].astype(np.int64)] = np.uint64(77 * 0x9E3779B97F4A7C15 % 2**64)
        out.append((o, l, i, v))
    return out


@pytest.mark.parametrize("V_dim", [10, 40])
def test_any_vdim_reproducible_on_sorted_path(V_dim):
    rng = np.random.default_rng(31 + V_dim)
    kw = dict(V_dim=V_dim, table_capacity=1 << 16, **dict(KW, V_threshold=1))
    batches = hot_batches(rng)
    A, B, G = capi.Engine(**kw), capi.Engine(**kw), capi.Engine(force_generic=1, **kw)
    A.profile(True)
    G.profile(True)
    for t in range(8):
        o, l, i, v = batches[t % len(batches)]
        is_train = t % 4 != 3
        pa, pb, pg = (X.train_step_raw(o, i, v, l, push_cnt=t < 2, is_train=is_train) for X in (A, B, G))
        assert pa.as_dict() == pb.as_dict(), f"step {t}"
        assert abs(pa.loss - pg.loss) <= 1e-4 * abs(pg.loss) + 1e-4, f"step {t}"
        assert abs(pa.penalty - pg.penalty) <= 1e-4 * abs(pg.penalty) + 1e-5, f"step {t}"
    keys = keys_of(batches)
    for a, b, g in zip(A.read_entries(keys), B.read_entries(keys), G.read_entries(keys)):
        assert np.array_equal(a, b)
        assert_close(a, g, what="sorted vs generic", **STATE_TOL)
    assert A.rng_state() == B.rng_state() == G.rng_state()
    assert (A.read_entries(keys)[1] == 1).sum() > 10
    # the CSC stage exists only on the sorted path (the generic one scatters with atomics)
    assert A.profile_read()["csc"]["count"] > 0
    assert G.profile_read()["csc"]["count"] == 0


# ---------------------------------------------------------------------------------------------------------------------
# 3. the pad columns of the last float4 are never updated
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [6, 10])
def test_pad_columns_stay_zero_with_v_lr_beta_0(V_dim):
    rng = np.random.default_rng(500 + V_dim)
    kw = dict(V_dim=V_dim, **dict(KW, V_lr_beta=0.0, V_threshold=1))
    batches = [rand_batch(rng, 128, 30, 300, j % 2 == 0) for j in range(4)]
    M, E = run_traj(kw, batches, epochs=3, raw=True)
    keys = keys_of(batches)
    ohasv = compare_state(M, E, keys)
    assert (ohasv == 1).sum() > 10
    for a in E.read_entries(keys):
        assert np.isfinite(a).all()
    ks = E.row_stride()
    assert ks == (V_dim + 3) // 4 * 4 and ks > V_dim
    dev = torch.device("cuda", 0)
    n = len(keys)
    d_keys = torch.from_numpy(keys.view(np.int64).copy()).to(dev)
    d_w = torch.zeros(n, dtype=torch.float32, device=dev)
    d_hasv = torch.zeros(n, dtype=torch.int32, device=dev)
    d_V = torch.full((n, ks), 7.0, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    E.dev_pull_rows(d_keys, n, d_w, d_hasv, d_V)
    E.sync()
    hasv, V = d_hasv.cpu().numpy(), d_V.cpu().numpy()
    rows = hasv == 1
    assert np.array_equal(rows, ohasv == 1)
    assert np.all(V[rows][:, V_dim:] == 0.0)
    assert np.array_equal(V[rows][:, :V_dim], E.read_entries(keys)[2][rows])


# ---------------------------------------------------------------------------------------------------------------------
# 4. a dropped raw batch (device-side key count) changes nothing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [10, 0])
def test_dropped_batch_changes_nothing(V_dim):
    id_bits = 30
    rng = np.random.default_rng(17 + V_dim)
    seq = idr.drop_batches(rng, id_bits, valued=True)
    kw = dict(V_dim=V_dim, id_bits=id_bits, table_capacity=1 << 14, **idr.KW)
    E, T = capi.Engine(**kw), capi.Engine(**kw)       # the twin never sees the bad batches
    keys = idr.seen_keys([b for _, b in seq])
    zero = (0.0,) * 4 + (0, 0)
    nbad = 0
    for t, (kind, (o, l, i, v)) in enumerate(seq):
        push = t < 3
        E.train_step_raw_async(len(l), o, i, v, l, push_cnt=push)
        rc, pr = idr.progress_rc(E, "dfb_wait_step")
        if kind == "bad":
            nbad += 1
            assert rc == capi.DFB_ERR_INVALID, f"step {t}: rc {rc}"
            assert "id_bits = %d" % id_bits in E.L.dfb_last_error(E.h).decode()
            assert idr.as_tuple(pr) == zero
            assert idr.as_tuple(E.read_progress()) == zero          # reported once
        else:
            assert rc == 0, f"step {t}: {E.L.dfb_last_error(E.h).decode()}"
            T.train_step_raw_async(len(l), o, i, v, l, push_cnt=push)
            rt, pt = idr.progress_rc(T, "dfb_wait_step")
            assert rt == 0 and idr.as_tuple(pr) == idr.as_tuple(pt), f"step {t}"
        idr.assert_same_model(E, T, keys)
    assert nbad == 2
    E.sync()
    assert idr.as_tuple(E.read_progress()) == zero


# ---------------------------------------------------------------------------------------------------------------------
# 5. the NVLink-sharded store, 1..3 ranks on one GPU
# ---------------------------------------------------------------------------------------------------------------------
SHARD_KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)
SHARD_STEPS = 7


def shard_train(step):
    return step % 3 != 2


def shard_batch(rank, step):
    """few distinct ids (every key held by several workers: the saved pull-time rows), binary / valued / empty
    batches in one step; a validation step re-reads the previous training step's ids"""
    src = step if shard_train(step) else step - 1
    if rank == 1 and step == 3:
        return raw_batch(rank, src, valued=False, B=0)
    return raw_batch(rank, src, valued=(rank + step) % 2 == 0, B=96, ids=60, max_nnz=24)


@pytest.mark.parametrize("V_dim", [0, 10, 40])
@pytest.mark.parametrize("S", [1, 2, 3])
def test_sharded_store_any_vdim_vs_simulation(S, V_dim):
    kw = dict(V_dim=V_dim, **SHARD_KW)
    engines, prog = run_local(S, kw, SHARD_STEPS, shard_batch, train_fn=shard_train)
    keys, own, shards = check_vs_simulation(engines, prog, kw, SHARD_STEPS, shard_batch, f"S={S} V_dim={V_dim}",
                                            train_fn=shard_train)
    if V_dim:
        assert sum((E.read_entries(keys[own == s])[1] == 1).sum() for s, E in enumerate(engines)) > 10
    for E in engines:
        E.close()


def test_sharded_store_one_rank_equals_fused_raw_step_v10():
    kw = dict(V_dim=10, **SHARD_KW)
    fn = lambda rank, step: raw_batch(rank, step, valued=(step % 2 == 0))     # noqa: E731
    engines, prog = run_local(1, kw, 6, fn)
    E2 = capi.Engine(device=0, table_capacity=1 << 14, **kw)
    for step in range(6):
        off, idx, val, lab = fn(0, step)
        pr2 = E2.train_step_raw(off, idx, val, lab, push_cnt=step < 2, is_train=True)
        assert abs(prog[0][step].loss - pr2.loss) <= 1e-5 * abs(pr2.loss) + 1e-5
        assert abs(prog[0][step].penalty - pr2.penalty) <= 1e-5 * abs(pr2.penalty) + 1e-6
    keys = all_keys(1, 6, fn)
    for a, b in zip(engines[0].read_entries(keys), E2.read_entries(keys)):
        assert_close(a, b, what="shard(S=1) vs fused raw step", rtol=1e-5, atol=1e-6)
    assert engines[0].rng_state() == E2.rng_state()


# ---------------------------------------------------------------------------------------------------------------------
# 6. the C++ CLI on 2 GPUs with criteo_sgd.conf's hyper-parameters (V_dim 10)
# ---------------------------------------------------------------------------------------------------------------------
def test_cli_two_gpus_criteo_sgd_conf(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import test_host_cpp as hc
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    hb.build()
    exe = os.path.join(hc.BIN, "difacto_b200")
    data, val = str(tmp_path / "train.libsvm"), str(tmp_path / "val.libsvm")
    hc._synthetic_libsvm(data, 8000, 1)
    hc._synthetic_libsvm(val, 1000, 2)
    conf = ["V_dim=10", "l1=10", "l2=10", "V_l2=10", "V_threshold=10", "lr=0.1", "V_lr=0.05"]
    common = [f"data_in={data}", f"data_val={val}", "batch_size=400", "shuffle=0", "num_jobs_per_epoch=1",
              "max_num_epochs=4", "stop_rel_objv=0", "stop_val_auc=-1e9", "table_capacity=65536"] + conf

    def losses(out, tag):
        return [float(x.split("loss = ")[1].split(",")[0]) for x in out.stdout.split("\n") if f"{tag}: loss" in x]

    one = subprocess.run([exe] + common, capture_output=True, text=True, timeout=300)
    assert one.returncode == 0, one.stderr[-2000:]
    model = str(tmp_path / "model")
    two = subprocess.run([exe] + common + ["num_gpus=2", f"model_out={model}"], capture_output=True, text=True,
                         timeout=300)
    assert two.returncode == 0, two.stderr[-2000:]
    t1, t2, v1, v2 = losses(one, "Training"), losses(two, "Training"), losses(one, "Validation"), losses(two, "Validation")
    assert len(t2) == 4 and len(v2) == 4
    assert t2[0] == pytest.approx(t1[0], rel=0.1)
    assert t2[-1] < t2[0]                                          # it learns
    assert v2[-1] == pytest.approx(v1[-1], rel=0.05)               # like the one-GPU run
    again = subprocess.run([exe, "task=predict", f"data_in={val}", f"model_in={model}", "num_gpus=2", "batch_size=400",
                            "table_capacity=65536"] + conf, capture_output=True, text=True, timeout=300)
    assert again.returncode == 0, again.stderr[-2000:]
    assert losses(again, "Prediction")[0] == pytest.approx(v2[-1], rel=1e-4)


# ---------------------------------------------------------------------------------------------------------------------
# 7. outside the range: V_dim 129
# ---------------------------------------------------------------------------------------------------------------------
def test_vdim_129_trains_on_generic_path_and_shard_init_refuses_it():
    rng = np.random.default_rng(129)
    kw = dict(V_dim=129, **dict(KW, V_threshold=1))
    batches = [rand_batch(rng, 96, 20, 200, j % 2 == 0) for j in range(3)]
    M, E = run_traj(kw, batches, epochs=2, raw=True)
    assert (compare_state(M, E, keys_of(batches)) == 1).sum() > 10
    S = capi.Engine(table_capacity=1 << 12, **kw)
    with pytest.raises(capi.DfbError):
        S.shard_init(0, 1, 128, 4096)
    assert "0..128" in S.L.dfb_last_error(S.h).decode()
