"""Checkpoints while training runs, and exact resume.

- dfb_snapshot_begin freezes the model on the device; dfb_frozen_write, on another thread while the engine keeps
  training, writes exactly what dfb_snapshot_write would have written at the moment of begin, and the engine trains
  exactly as its twin that took a blocking snapshot (V_dim 0 / 10 / 64, binary and valued, a growing engine that
  rehashes during the write, three sharded ranks on one GPU).
- A write_fn that fails mid-stream fails the write only.
- dfb_id_range_set: an engine given a learned id range sorts and drops batches as the one that learned it.
- The CLI: checkpoint_out / checkpoint_period / checkpoint_in resume a run that ended mid-part, and the resumed run
  prints the epochs and saves the model of the uninterrupted run, byte for byte; mismatched settings and a pointer to
  a missing checkpoint are refused, stale files of a later checkpoint ignored.
"""
import ctypes as C
import os
import struct
import subprocess
import sys
import threading

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # several engines on one GPU: one hardware queue per stream

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from shard_sim import raw_batch, run_local  # noqa: E402

pytestmark = pytest.mark.gpu
capi = pytest.importorskip("difacto_b200.capi")

KW = dict(l1=0.05, l2=0.01, lr=0.2, V_lr=0.1, V_threshold=1, V_l2=0.01, V_init_scale=0.2, seed=3)
PROGRESS = ("loss", "penalty", "auc", "nrows", "new_keys", "new_vrows")


class Sink:
    def __init__(self, fail_after=None):
        self.parts, self.n, self.fail_after = [], 0, fail_after

    def write(self, b):
        if self.fail_after is not None and self.n + len(b) > self.fail_after:
            raise IOError("disk full")
        self.parts.append(bytes(b))
        self.n += len(b)

    def value(self):
        return b"".join(self.parts)


def as_tuple(pr):
    return tuple(getattr(pr, f) for f in PROGRESS)


def step(E, b, j):
    off, idx, val, lab = b
    pr, pred = E.train_step_raw(off, idx, val, lab, push_cnt=j < 2, is_train=True, want_pred=True)
    return as_tuple(pr), pred


def blocking(E, chunk=0):
    s = Sink()
    E.snapshot_to(s, chunk_bytes=chunk)
    return s.value()


def frozen_while_training(A, B, batches, t, chunk):
    """A and B train batches[:t]; then A freezes and B writes a blocking snapshot; both train the rest while A's copy
    is written on another thread.  Returns A's bytes and B's."""
    for j in range(t):
        assert step(A, batches[j], j)[0] == step(B, batches[j], j)[0]
    f = A.snapshot_begin()
    want = blocking(B)
    sink, err = Sink(), []

    def write():
        try:
            f.write_to(sink, chunk_bytes=chunk)
        except Exception as e:      # surfaced below
            err.append(e)
    th = threading.Thread(target=write)
    th.start()
    for j in range(t, len(batches)):
        (pa, qa), (pb, qb) = step(A, batches[j], j), step(B, batches[j], j)
        assert pa == pb and np.array_equal(qa, qb), f"step {j}"
    th.join()
    assert not err, err
    f.release()
    assert blocking(A) == blocking(B)
    return sink.value(), want


@pytest.mark.parametrize("V_dim", [0, 10, 64])
@pytest.mark.parametrize("valued", [False, True])
def test_frozen_write_equals_the_blocking_write(V_dim, valued):
    batches = [raw_batch(0, j, valued, B=200, ids=4000, max_nnz=30, seed=V_dim) for j in range(10)]
    A = capi.Engine(V_dim=V_dim, table_capacity=1 << 15, **KW)
    B = capi.Engine(V_dim=V_dim, table_capacity=1 << 15, **KW)
    got, want = frozen_while_training(A, B, batches, 4, chunk=4096)
    assert len(want) > 40 and got == want
    # one frozen snapshot per handle
    f = A.snapshot_begin()
    with pytest.raises(capi.DfbError):
        A.snapshot_begin()
    f.release()
    A.snapshot_begin().release()
    # a copy left behind is freed with the engine; its wrapper then refuses to write and releases nothing
    f = A.snapshot_begin()
    A.close()
    with pytest.raises(capi.DfbError, match="released"):
        f.write_to(Sink())
    f.release()


def test_frozen_write_outlives_a_rehash():
    """a growing engine rehashes into a new table while the copy of the old one is written"""
    kw = dict(KW, V_dim=16, table_capacity=1024, table_capacity_max=1 << 18)
    batches = [raw_batch(0, j, True, B=300, ids=1 << 20, max_nnz=30, seed=5) for j in range(10)]
    A, B = capi.Engine(**kw), capi.Engine(**kw)
    for j in range(2):
        step(A, batches[j], j), step(B, batches[j], j)
    cap0 = A.table_stats()["capacity"]
    got, want = frozen_while_training(A, B, batches[2:], 0, chunk=2048)
    assert A.table_stats()["capacity"] > cap0, "the engine must have grown during the write"
    assert got == want


def test_frozen_write_of_sharded_ranks():
    """3 ranks of the sharded store on one GPU: each rank's frozen part equals its twin rank's blocking part"""
    S, kw = 3, dict(KW, V_dim=16)
    fn = lambda r, s: raw_batch(r, s, s % 2 == 0, seed=9)   # noqa: E731
    A, pa = run_local(S, kw, 4, fn)
    B, pb = run_local(S, kw, 4, fn)
    assert [[as_tuple(p) for p in x] for x in pa] == [[as_tuple(p) for p in x] for x in pb]
    frozen = [E.snapshot_begin() for E in A]
    want = [blocking(E) for E in B]
    sinks = [Sink() for _ in range(S)]
    th = [threading.Thread(target=f.write_to, args=(s, 4096)) for f, s in zip(frozen, sinks)]
    for t in th:
        t.start()
    _, pa = run_local(S, kw, 4, lambda r, s: fn(r, s + 4), engines=A, cnt_steps=0)
    _, pb = run_local(S, kw, 4, lambda r, s: fn(r, s + 4), engines=B, cnt_steps=0)
    for t in th:
        t.join()
    assert [[as_tuple(p) for p in x] for x in pa] == [[as_tuple(p) for p in x] for x in pb]
    for r in range(S):
        assert sinks[r].value() == want[r], f"rank {r}"
        frozen[r].release()


def test_a_failing_sink_fails_the_write_only():
    batches = [raw_batch(0, j, True, B=200, ids=3000, max_nnz=30, seed=2) for j in range(8)]
    A = capi.Engine(V_dim=10, table_capacity=1 << 14, **KW)
    B = capi.Engine(V_dim=10, table_capacity=1 << 14, **KW)
    for j in range(4):
        assert step(A, batches[j], j)[0] == step(B, batches[j], j)[0]
    f = A.snapshot_begin()
    with pytest.raises(capi.DfbError, match="sink failed"):
        f.write_to(Sink(fail_after=10000), chunk_bytes=1024)
    s = Sink()
    f.write_to(s, chunk_bytes=1024)          # the copy is still whole: a second write succeeds
    assert s.value() == blocking(B)
    f.release()
    for j in range(4, 8):
        (pa, qa), (pb, qb) = step(A, batches[j], j), step(B, batches[j], j)
        assert pa == pb and np.array_equal(qa, qb)
    assert blocking(A) == blocking(B)


# ---------------------------------------------------------------------------------------------------------------------
# the learned id range
# ---------------------------------------------------------------------------------------------------------------------
def id_batch(rng, bits, B=120):
    lens = rng.integers(1, 20, B)
    n = int(lens.sum())
    ids = rng.integers(0, 1 << min(bits, 62), n, dtype=np.uint64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    lab = np.where(rng.random(B) < 0.4, 1.0, -1.0).astype(np.float32)
    return off, ids, None, lab


def async_steps(E, batches):
    out = []
    for off, ids, val, lab in batches:
        E.train_step_raw_async(len(lab), off, ids, val, lab)
        pr = capi.Progress()
        rc = E.L.dfb_wait_step(E.h, C.byref(pr))
        E.sync()                      # the batch's key mask is back before the next batch is localized
        out.append((rc, as_tuple(pr) if rc == 0 else None))
    return out


def test_a_given_id_range_trains_and_drops_as_the_learned_one():
    rng = np.random.default_rng(4)
    first = id_batch(rng, 20)
    later = [id_batch(rng, b) for b in (18, 40, 20, 44, 19)]
    L = capi.Engine(V_dim=8, table_capacity=1 << 15, **KW)
    assert L.id_range() == 0
    async_steps(L, [first])
    bits = L.id_range()
    assert 0 < bits <= 24          # ids below 2^20: the byte-reversed keys have no bit set below bit 40
    G = capi.Engine(V_dim=8, table_capacity=1 << 15, **KW)
    G.set_id_range(bits)
    assert G.id_range() == bits
    with pytest.raises(capi.DfbError):
        G.set_id_range(bits)           # only on an engine without a range
    # the model of L's first batch, then the same batches on both: the same drops, the same Progress
    buf = Sink()
    L.snapshot_to(buf)
    G.restore(buf.value())
    rl, rg = async_steps(L, later), async_steps(G, later)
    assert rl == rg
    assert any(rc != 0 for rc, _ in rl), "some batch must fall outside the learned range"
    assert L.id_range() == G.id_range()
    assert blocking(L) == blocking(G)


# ---------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def exe():
    from difacto_b200 import build as eb
    from difacto_b200.host import build as hb
    eb.build()
    hb.build()
    return os.path.join(ROOT, "difacto_b200", "host", "bin", "difacto_b200")


def write_libsvm(path, rows, seed):
    rng = np.random.default_rng(seed)
    with open(path, "w") as f:
        for _ in range(rows):
            ids = np.unique(rng.zipf(1.3, int(rng.integers(1, 25))) % 5000)
            vals = rng.random(len(ids)).astype(np.float32) + 0.1
            f.write(("1 " if rng.random() < 0.3 else "-1 ") + " ".join(f"{i}:{v:.9g}" for i, v in zip(ids, vals)) + "\n")


def epoch_lines(out, first):
    lines = [l for l in out.split("\n") if l.startswith(("Start epoch", " - Training", " - Validation"))]
    i = lines.index(f"Start epoch {first}")
    return lines[i:]


def checkpoint_lines(out):
    """minibatch -> (epoch, [(part, minibatches read from it) per worker]) of the learner's checkpoint lines"""
    at = {}
    for line in out.split("\n"):
        if line.startswith("Checkpoint "):
            head, pairs = line.split(", part:minibatches ")
            m = int(head.split("minibatch ")[1].split(",")[0])
            at[m] = (int(head.split("epoch ")[1]), [tuple(int(x) for x in w.split(":")) for w in pairs.split()])
    return at


def read_state(path):
    """the epoch and the workers' {part, consumed} of a checkpoint state record"""
    b = open(path, "rb").read()
    assert b[:8] == b"DFBCKST\x00"
    p = 12
    (ns,) = struct.unpack_from("<I", b, p)
    p += 4
    for _ in range(2 * ns):
        (n,) = struct.unpack_from("<I", b, p)
        p += 4 + n
    epoch, nw = struct.unpack_from("<iI", b, p)
    p += 8
    return epoch, [struct.unpack_from("<iQ", b, p + 12 * i) for i in range(nw)]


def run(exe, args):
    return subprocess.run([exe] + args, capture_output=True, text=True, timeout=600)


def resume_case(exe, tmp_path, num_gpus):
    data, val = str(tmp_path / "train.libsvm"), str(tmp_path / "val.libsvm")
    write_libsvm(data, 1200, 1)
    write_libsvm(val, 300, 2)
    E = 2
    common = [f"data_in={data}", f"data_val={val}", "V_dim=16", "l1=0.05", "lr=0.2", "V_threshold=2",
              "batch_size=50", "shuffle=2", "neg_sampling=0.5", "num_jobs_per_epoch=3", "stop_rel_objv=0",
              "table_capacity=65536", f"num_gpus={num_gpus}"]
    P = str(tmp_path / "ckpt")
    C_ = run(exe, common + [f"max_num_epochs={E + 1}", f"model_out={tmp_path / 'c.model'}"])
    assert C_.returncode == 0, C_.stderr[-2000:]
    # a checkpoint after every minibatch shows where each one falls (checkpoints change nothing about the run); pick the
    # period whose last checkpoint in the run of E epochs falls inside a part, and not at its end
    every = run(exe, common + [f"max_num_epochs={E}", f"checkpoint_out={tmp_path / 'every'}", "checkpoint_period=1"])
    assert every.returncode == 0, every.stderr[-2000:]
    at = checkpoint_lines(every.stdout)               # minibatch -> (epoch, [(part, consumed) per worker])
    part_len = {}
    for ep, ws in at.values():
        for r, (part, k) in enumerate(ws):
            part_len[(ep, r, part)] = max(part_len.get((ep, r, part), 0), k)
    total = max(at)

    def mid_part(m):
        ep, ws = at[m]
        return ep == E - 1 and any(0 < k < part_len[(ep, r, part)] for r, (part, k) in enumerate(ws))
    period = next(p for p in range(5, total) if mid_part(total // p * p))
    A = run(exe, common + [f"max_num_epochs={E}", f"checkpoint_out={P}", f"checkpoint_period={period}"])
    assert A.returncode == 0, A.stderr[-2000:]
    assert epoch_lines(A.stdout, 0) == epoch_lines(every.stdout, 0)
    c = int(open(P).read())
    assert c == total // period - 1
    assert not os.path.exists(f"{P}.{c - 1}.state"), "the previous checkpoint is removed"
    epoch, workers = read_state(f"{P}.{c}.state")
    assert (epoch, [tuple(w) for w in workers]) == at[total // period * period]
    # stale files of a later checkpoint, as a crash before the pointer's rename leaves them, are ignored
    for suffix in (".state", ".model", ".model_part-0", ".model_part-1"):
        open(f"{P}.{c + 1}{suffix}", "wb").write(b"stale")
    # the same settings spelled otherwise, and defaults given explicitly, are the same settings
    B = run(exe, common + [f"max_num_epochs={E + 1}", f"checkpoint_in={P}", f"model_out={tmp_path / 'b.model'}",
                           "l1=0.050", "seed=0", "lr_beta=1.0", "V_threshold=+2"])
    assert B.returncode == 0, B.stderr[-2000:]
    assert "Resuming from checkpoint" in B.stdout
    assert epoch_lines(B.stdout, epoch) == epoch_lines(C_.stdout, epoch)
    for r in range(num_gpus):
        name = (lambda b: f"{b}_part-{r}") if num_gpus > 1 else (lambda b: b)
        assert open(name(tmp_path / "b.model"), "rb").read() == open(name(tmp_path / "c.model"), "rb").read()
    return common, P, c


def test_cli_resume_one_gpu(exe, tmp_path):
    common, P, c = resume_case(exe, tmp_path, 1)
    # refusals: another batch_size; a pointer to a checkpoint that is not there
    bad = run(exe, [a for a in common if not a.startswith("batch_size")] + ["batch_size=64", f"checkpoint_in={P}"])
    assert bad.returncode != 0 and "batch_size" in bad.stderr
    bad = run(exe, common + ["seed=4294967295", f"checkpoint_in={P}"])
    assert bad.returncode != 0 and "seed" in bad.stderr
    missing = str(tmp_path / "missing")
    open(missing, "w").write("999\n")
    bad = run(exe, common + [f"checkpoint_in={missing}"])
    assert bad.returncode != 0 and "missing" in bad.stderr


def test_cli_resume_two_gpus(exe, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    resume_case(exe, tmp_path, 2)
