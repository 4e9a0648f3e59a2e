"""GPU localizer on batches that span many tiles of its single-pass emit (2048 sorted pairs per tile), with key runs
that cross tile boundaries, including one key present in every row: the raw-id step on device-resident batches must
stay bit-identical to the host-localized step.  Host offsets that run backwards are rejected."""
import numpy as np
import pytest

from oracle import oracle as O
from util import localized

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")
torch = pytest.importorskip("torch")


def tiled_batch(rng, B, id_space, mult, valued):
    """rows of 1..40 ids over a small id space (runs of ~100 pairs per key after the sort) plus the id 0 in every row
    (one run of B pairs)"""
    nnzr = rng.integers(0, 40, B) + 1
    off = np.concatenate([[0], np.cumsum(nnzr)]).astype(np.uint64)
    n = int(off[-1])
    idx = (rng.integers(1, id_space, n).astype(np.uint64) * np.uint64(mult))
    idx[(off[:-1] + rng.integers(0, nnzr)).astype(np.int64)] = 0
    val = (rng.random(n).astype(np.float32) * 2 - 0.5) if valued else None
    lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, lab, idx, val


@pytest.mark.parametrize("mult,valued", [(1, False), (0x9E3779B97F4A7C15, True)])    # 32-bit and 64-bit sort keys
def test_raw_dev_step_many_emit_tiles_equals_localized_step(mult, valued):
    rng = np.random.default_rng(11)
    kw = dict(V_dim=16, l1=0.2, l2=0.01, lr=0.2, V_lr=0.05, V_threshold=3, V_l2=0.02, V_init_scale=0.2, seed=5)
    batches = [tiled_batch(rng, 3000, 500, mult, valued and j % 2 == 0) for j in range(3)]
    assert all(int(b[0][-1]) > 20 * 2048 for b in batches)
    R = capi.Engine(table_capacity=1 << 14, **kw)     # raw ids on the device -> GPU localizer, no sync between steps
    L = capi.Engine(table_capacity=1 << 14, **kw)     # host-localized
    dev = torch.device("cuda", 0)
    devb = [tuple(None if a is None else torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).to(dev)
                  for a in b) for b in batches]
    loss_l = 0.0
    for ep in range(3):
        for (o, l, i, v), (do, dl, di, dv) in zip(batches, devb):
            R.train_step_raw_dev(len(l), len(i), do, di, dv, dl, ep == 0, True)
            b = localized((o, l, i, v))
            loss_l += L.train_step(o, b["lidx"], v, l, b["keys"], b["cnt"] if ep == 0 else None, True).loss
    R.sync()
    loss_r = R.read_progress().loss
    assert abs(loss_r - loss_l) <= 1e-6 * abs(loss_l)     # summed on the device vs per step on the host
    for (o, l, i, v) in batches:          # the localizer's own outputs on the same batches
        gl, gk, gc = R.localize(o, i)
        ol, ok, oc = O.localize(o, i)
        assert np.array_equal(gl, ol) and np.array_equal(gk, ok) and np.array_equal(gc, oc)
    keys = np.unique(np.concatenate([O.reverse_bytes_np(b[2]) for b in batches]))
    for a, b in zip(R.read_entries(keys), L.read_entries(keys)):
        assert np.array_equal(a, b)        # same kernels, same CSC order: bit-identical


def test_localize_rejects_decreasing_offsets():
    E = capi.Engine(V_dim=0, table_capacity=1 << 10)
    off = np.array([0, 5, 3, 8], np.uint64)          # row 1 runs backwards
    with pytest.raises(capi.DfbError):
        E.localize(off, np.arange(8, dtype=np.uint64))
    lidx, keys, cnt = E.localize(np.array([0, 5, 5, 8], np.uint64), np.arange(8, dtype=np.uint64))   # empty row: fine
    assert len(lidx) == 8 and len(keys) == 8
