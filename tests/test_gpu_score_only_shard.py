"""Scoring-only ranks of the fused sharded store (score_only = 1, V_storage = fp32 | bf16, dfb_shard_init).

Pinned here: a store of fp32 scoring ranks gives, bit for bit, the predictions and Progress of the training store whose
snapshots it restored (the owners run the same partial-sum kernel at the V-only row stride); bf16 scoring ranks give,
bit for bit, what fp32 scoring ranks give on the model rounded to bf16 beforehand, and stay within the bf16 bound of one
engine holding the unrounded model, also after M = 2 parts were restored into N = 3 growing ranks; training and scoring
ranks mix in one store; every step that trains, counts features or validates is refused by name on a scoring rank
before anything is enqueued; the CLI scores a num_gpus = 2 model on two scoring ranks."""
import functools
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from shard_sim import raw_batch, run_local

import test_gpu_id_range as idr
from test_gpu_checkpoint import restore_parts
from test_gpu_score_only import rounded

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")

KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=2, V_l2=0.02, V_init_scale=0.2, seed=11, hot_split=64)
ENGINE = dict(table_capacity=1 << 14, shard_timeout_ms=8000)
SHAPE = dict(max_rows=128, max_nnz=16384)
VDIMS = [0, 5, 10, 16, 64, 100, 128]
B = 96


def batches(S, step, valued):
    """one predict batch per rank: mixed row lengths (empty, one chunk, several, 1024..1500 nonzeros), over ids of which
    a third are not in the model"""
    return [raw_batch(r, step, valued, ids=900, mixed=True, B=B) for r in range(S)]


def predict(engines, bs):
    """one predict step of every rank (rank 0 of a multi-rank store without labels): [(Progress, prediction bytes)]"""
    S = len(engines)
    outs = [torch.zeros(B, dtype=torch.float32, pin_memory=True) for _ in range(S)]
    for r, (E, (off, ids, val, lab)) in enumerate(zip(engines, bs)):
        E.shard_begin_predict_async(len(lab), off, ids, val, None if (r == 0 and S > 1) else lab, outs[r])
    for ph in range(5):
        for E in engines:
            E.shard_phase(ph)
    return [(idr.as_tuple(E.wait_step()), outs[r].numpy().tobytes()) for r, E in enumerate(engines)]


def kind_kw(kind):
    return {} if kind is None else dict(score_only=1, V_storage=kind)


def store(V_dim, kinds, blobs, **ekw):
    """len(kinds) ranks of one GPU (kind None: training layout, "fp32" / "bf16": scoring), connected, then each rank r
    restores blobs[r] -- after dfb_shard_init, as the CLI does"""
    engines = [capi.Engine(V_dim=V_dim, **{**KW, **ENGINE, **ekw, **kind_kw(k)}) for k in kinds]
    from difacto_b200.sharded import FusedShardedStore
    FusedShardedStore.connect_local(engines, **SHAPE)
    for E, blob in zip(engines, blobs):
        if blob is not None:
            E.restore(blob)
    return engines


@functools.lru_cache(maxsize=None)
def trained(S, V_dim):
    """S training ranks after 4 steps (binary and valued batches): each rank's snapshot, and the predict steps of that
    training store on the binary and the valued predict batches"""
    fn = lambda r, st: raw_batch(r, st, valued=(st % 2 == 0), ids=600, mixed=True, B=B)   # noqa: E731
    engines, _ = run_local(S, dict(KW, V_dim=V_dim), 4, fn, **SHAPE)
    want = {valued: predict(engines, batches(S, 10 + valued, valued)) for valued in (False, True)}
    snaps = tuple(E.snapshot() for E in engines)
    if V_dim:
        assert sum(E.table_stats()["n_vrows"] for E in engines) > 100
    for E in engines:
        E.close()
    return snaps, want


def check_predict_progress(res, S):
    for r, (pr, q) in enumerate(res):
        loss, penalty, auc, nrows, new_keys, new_vrows = pr
        assert nrows == B and penalty == 0 and new_keys == 0 and new_vrows == 0, (r, pr)
        if r == 0 and S > 1:
            assert loss == 0 and auc == 0
        assert np.frombuffer(q, np.float32).any()


# ---------------------------------------------------------------------------------------------------------------------
# 1. fp32 scoring ranks = the training ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", VDIMS)
@pytest.mark.parametrize("S", [2, 3])
def test_fp32_scoring_shards_are_bitwise_the_training_shards(S, V_dim):
    snaps, want = trained(S, V_dim)
    F = store(V_dim, ["fp32"] * S, snaps)
    assert [E.row_bytes()[0] for E in F] == [4 * ((V_dim + 3) // 4 * 4)] * S
    for valued in (False, True):
        got = predict(F, batches(S, 10 + valued, valued))
        check_predict_progress(got, S)
        assert got == want[valued], (S, V_dim, valued)


# ---------------------------------------------------------------------------------------------------------------------
# 2. bf16 scoring ranks = fp32 scoring ranks of the rounded model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", VDIMS)
@pytest.mark.parametrize("S", [2, 3])
def test_bf16_scoring_shards_are_bitwise_fp32_shards_of_the_rounded_model(S, V_dim):
    snaps, want = trained(S, V_dim)
    pre = [rounded(b, V_dim) if V_dim else b for b in snaps]
    H = store(V_dim, ["bf16"] * S, snaps)
    F = store(V_dim, ["fp32"] * S, pre)
    for valued in (False, True):
        bs = batches(S, 10 + valued, valued)
        got = predict(H, bs)
        check_predict_progress(got, S)
        assert got == predict(F, bs), (S, V_dim, valued)
        if V_dim >= 10:                                  # and rounding did change a prediction
            assert [q for _, q in got] != [q for _, q in want[valued]]


# ---------------------------------------------------------------------------------------------------------------------
# 3. bf16 scoring ranks against one engine holding the unrounded model; 2 parts into 3 growing ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [10, 64, 128])
def test_two_parts_into_three_growing_bf16_ranks_are_close_to_one_engine(V_dim):
    """The bound of test_gpu_score_only.test_bf16_scoring_is_close_to_the_oracle: rounding V to bf16 moves a score by
    at most (2^-8 + 2^-18) S, S = sum_{i<j} |x_i x_j| <|V_i|, |V_j|>; allowed: 2^-7 S, plus 1e-4 (1 + |score|) for the
    fp32 sums, which the store adds up owner by owner."""
    parts, _ = trained(2, V_dim)
    one = capi.Engine(V_dim=V_dim, table_capacity=1 << 15, **KW)           # training layout: read_entries gives V
    restore_parts([one], list(parts))
    grow = store(V_dim, ["bf16"] * 3, [None] * 3, table_capacity=32, table_capacity_max=1 << 20)
    restore_parts(grow, list(parts))
    st = [g.table_stats() for g in grow]
    assert sum(s["n_keys"] for s in st) == one.table_stats()["n_keys"]
    assert sum(s["n_vrows"] for s in st) == one.table_stats()["n_vrows"]
    assert min(s["capacity"] for s in st) > 32 and min(s["v_capacity"] for s in st) > 32, st
    for valued in (False, True):
        bs = batches(3, 20 + valued, valued)
        got = predict(grow, bs)
        check_predict_progress(got, 3)
        for r, (off, ids, val, lab) in enumerate(bs):
            _, want = one.predict_raw(off, ids, val, lab)
            g = np.frombuffer(got[r][1], np.float32)
            lidx, keys, _ = O.localize(off, ids)
            _, hasv, V, _ = one.read_entries(keys)
            absV = np.where((hasv == 1)[:, None], np.abs(V.astype(np.float64)), 0.0)
            x = np.ones(len(ids)) if val is None else np.abs(val.astype(np.float64))
            for i in range(len(lab)):
                a, e = int(off[i]), int(off[i + 1])
                rows = x[a:e, None] * absV[lidx[a:e]]
                Sij = 0.5 * ((rows.sum(0) ** 2).sum() - (rows ** 2).sum())
                assert abs(float(g[i]) - float(want[i])) <= 2.0 ** -7 * Sij + 1e-4 * (1 + abs(float(want[i]))), \
                    (V_dim, valued, r, i, Sij)


# ---------------------------------------------------------------------------------------------------------------------
# 4. training and scoring ranks in one store
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V_dim", [10, 64])
def test_a_store_mixes_training_fp32_and_bf16_ranks(V_dim):
    snaps, want = trained(3, V_dim)
    mixed = store(V_dim, [None, "fp32", "bf16"], snaps)
    ref = store(V_dim, ["fp32"] * 3, [snaps[0], snaps[1], rounded(snaps[2], V_dim)])
    for valued in (False, True):
        bs = batches(3, 10 + valued, valued)
        got = predict(mixed, bs)
        assert got == predict(ref, bs)
        assert got != want[valued]                       # rank 2's rounding reaches every worker's rows


# ---------------------------------------------------------------------------------------------------------------------
# 5. refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "bf16"])
def test_a_scoring_rank_refuses_every_step_but_predict(storage):
    S, V_dim = 2, 16
    snaps, want = trained(S, V_dim)
    E = store(V_dim, [storage] * S, snaps)
    bs = batches(S, 11, True)
    before = predict(E, bs)
    if storage == "fp32":
        assert before == want[True]
    for r, R in enumerate(E):
        off, ids, val, lab = bs[r]
        calls = {}
        for train in (True, False):
            calls.update({      # (train False: a validation step)
                f"shard_step_async {train}": lambda t=train: R.shard_step_async(B, off, ids, val, lab, t, t),
                f"shard_begin_async {train}": lambda t=train: R.shard_begin_async(B, off, ids, val, lab, t, t),
                f"shard_step_dev {train}": lambda t=train: R.shard_step_dev(0, 0, None, None, None, None, t, t),
                f"shard_begin_dev {train}": lambda t=train: R.shard_begin_dev(0, 0, None, None, None, None, t, t),
            })
        for name, call in calls.items():
            with pytest.raises(capi.DfbError) as e:
                call()
            assert e.value.code == capi.DFB_ERR_INVALID and "score_only" in str(e.value), (r, name, str(e.value))
        with pytest.raises(capi.DfbError) as e:
            R.shard_init(r, S, 128, 4096)
        assert e.value.code == capi.DFB_ERR_INVALID and "already" in str(e.value)
    assert predict(E, bs) == before                     # nothing was enqueued: no rank waits for a step of another
    assert E[0].shard_info()["steps"] == 2


def test_shard_init_on_a_training_engine_refuses_what_it_refused():
    for kw in (dict(table_capacity=1024, table_capacity_max=1 << 20), dict(force_generic=1), dict(scatter="atomic")):
        E = capi.Engine(V_dim=16, **KW, **kw)
        with pytest.raises(capi.DfbError) as e:
            E.shard_init(0, 1, 128, 4096)
        assert e.value.code == capi.DFB_ERR_INVALID, kw
    # a growing scoring rank is accepted: its predict steps never insert.  A one-rank store of a scoring engine is not:
    # on its own the engine scores with predict_raw*
    G = capi.Engine(V_dim=16, table_capacity=1024, table_capacity_max=1 << 20, score_only=1)
    with pytest.raises(capi.DfbError) as e:
        G.shard_init(0, 1, 128, 4096)
    assert e.value.code == capi.DFB_ERR_INVALID and "score_only" in str(e.value)
    G.shard_init(0, 2, 128, 4096)


# ---------------------------------------------------------------------------------------------------------------------
# 6. CLI: task=predict num_gpus=2 score_only=1
# ---------------------------------------------------------------------------------------------------------------------
def test_cli_scores_a_two_gpu_model_on_two_scoring_ranks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from test_gpu_checkpoint import cli_kw, read_libsvm, write_libsvm
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    exe = os.path.join(hb.build(), "difacto_b200")
    data, model = str(tmp_path / "d.libsvm"), str(tmp_path / "m")
    write_libsvm(data, 3000, 17)
    off, idx, val, lab = read_libsvm(data)
    common = [f"data_in={data}"] + cli_kw()
    out = subprocess.run([exe] + common + ["max_num_epochs=2", "num_gpus=2", f"model_out={model}"], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]

    def run(extra, name=None):
        po = [f"pred_out={tmp_path / name}"] if name else []
        o = subprocess.run([exe] + common + ["task=predict", "num_gpus=2", f"model_in={model}"] + po + extra,
                           capture_output=True, text=True, timeout=600)
        assert o.returncode == 0, (extra, o.stderr[-2000:])
        assert "unrecognized" not in o.stderr
        return o.stdout.split("Prediction: ")[1].split("\n")[0], (open(tmp_path / name, "rb").read() if name else None)

    _, want = run([], "p0")
    line, got = run(["score_only=1"], "p1")
    assert got == want
    _, got16 = run(["score_only=1", "V_storage=bf16"], "p2")
    p, q = np.loadtxt(want.decode().split(), dtype=np.float32), np.loadtxt(got16.decode().split(), dtype=np.float32)
    assert p.shape == q.shape == (3000,) and got16 != want
    # the bound of test_bf16_scoring_is_close_to_the_oracle with |V| <= vmax, |x| <= 1.25 and at most 29 nonzeros a
    # row: S <= C(29, 2) 1.25^2 V_dim vmax^2.  vmax: of the model the ranks saved
    T = capi.Engine(V_dim=16, table_capacity=1 << 14)
    restore_parts([T], [open(f"{model}_part-{r}", "rb").read() for r in range(2)])
    vmax = float(np.abs(T.read_entries(np.unique(O.reverse_bytes_np(idx.copy())))[2]).max())
    assert vmax > 0 and np.abs(p - q).max() <= 2.0 ** -7 * 406 * 1.5625 * 16 * vmax * vmax + 1e-3
    # without pred_out: predict steps all the same (a validation step would be refused by the scoring ranks)
    assert run(["score_only=1"])[0] == line
