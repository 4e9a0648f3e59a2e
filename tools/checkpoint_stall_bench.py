"""How long a checkpoint stops training: the blocking write (dfb_snapshot_write) against a frozen device copy
(dfb_snapshot_begin) written by another thread (dfb_frozen_write) while the engine keeps training.

    python tools/checkpoint_stall_bench.py [--batches 8] [--window 20] [--out DIR]

The engine is filled as tools/checkpoint_bench.py fills it (raw minibatches of 65536 rows x 100 binary ids, V_dim 64,
every key with a V row; 8 batches ~ 52 M keys).  Then windows of `window` steps, each with one checkpoint in the
middle, over four cached minibatches whose keys are already in the table (the table does not grow).  The sinks are C
functions (compiled into a temporary directory at start), as the C++ learner's are: one that discards and one that
write()s to a file in the temporary directory (unlinked; skipped without room for the snapshot).  The writer thread
never takes the interpreter lock, so the steps of the main thread see only what the GPU and the host share.
Per mode and sink:
  * stall_ms: the time from the checkpoint call until the engine may train again; for the frozen copy split into
    drain_ms (waiting for the engine's streams) and begin_ms (allocating and mapping the copy's memory, and the copy,
    whose time at the card's device-to-device copy rate is copy_ms_est);
  * the steps before the checkpoint and those that ran while the write ran: count, median and mean step time, and
    steps_during_frac = steps per second during the write / steps per second before;
  * write_s: the time of the whole write.
Prints one JSON line (and writes it to DIR/checkpoint_stall_bench.json with --out).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from checkpoint_bench import IDS, NNZ, ROWS, filled_engine  # noqa: E402
from difacto_b200 import capi  # noqa: E402

SINKS_C = r"""
#include <errno.h>
#include <stddef.h>
#include <unistd.h>
int sink_discard(void* ctx, const void* buf, size_t n) { (void)ctx; (void)buf; (void)n; return 0; }
int sink_fd(void* ctx, const void* buf, size_t n) {
  const int fd = *(const int*)ctx;
  const char* p = (const char*)buf;
  while (n) {
    const ssize_t w = write(fd, p, n);
    if (w < 0) { if (errno == EINTR) continue; return 1; }
    p += w; n -= (size_t)w;
  }
  return 0;
}
"""


def c_sinks(tmpdir):
    src, so = os.path.join(tmpdir, "sinks.c"), os.path.join(tmpdir, "sinks.so")
    with open(src, "w") as f:
        f.write(SINKS_C)
    subprocess.run(["cc", "-O2", "-shared", "-fPIC", "-o", so, src], check=True)
    lib = C.CDLL(so)
    addr = lambda fn: C.cast(fn, C.c_void_p).value   # noqa: E731
    return capi.WRITE_FN(addr(lib.sink_discard)), capi.WRITE_FN(addr(lib.sink_fd))


def d2d_gbps():
    n = 2 << 30
    a = torch.empty(n, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    b.copy_(a)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        b.copy_(a)
    torch.cuda.synchronize()
    gbps = 5 * n / (time.perf_counter() - t0) / 1e9
    del a, b
    torch.cuda.empty_cache()
    return gbps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--window", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    E = filled_engine(a.batches, seed=1)
    g = torch.Generator(device="cuda").manual_seed(7)
    off = torch.arange(ROWS + 1, device="cuda", dtype=torch.int64) * NNZ
    lab = torch.where(torch.rand(ROWS, device="cuda", generator=g) < 0.3, 1.0, -1.0)
    cached = [torch.randint(0, IDS, (ROWS * NNZ,), device="cuda", generator=g, dtype=torch.int64) for _ in range(4)]
    t = [0]

    def step():
        E.train_step_raw_dev(ROWS, ROWS * NNZ, off, cached[t[0] % 4], None, lab, False, True)
        t[0] += 1
        E.sync()

    for _ in range(8):      # the cached batches' keys are inserted here, once
        step()
    st = E.table_stats()
    res = dict(bench="checkpoint_stall", n_keys=st["n_keys"], n_vrows=st["n_vrows"], window=a.window)

    def timed_step():
        t0 = time.perf_counter()
        step()
        return (time.perf_counter() - t0) * 1e3

    def stats(ms):
        return dict(n=len(ms), median_ms=round(statistics.median(ms), 3), mean_ms=round(statistics.mean(ms), 3),
                    total_s=round(sum(ms) / 1e3, 3)) if ms else None

    def window(mode, fn, fd):
        ctx = C.c_int(fd)
        before = [timed_step() for _ in range(a.window // 2)]
        t0 = time.perf_counter()
        r = {}
        if mode == "blocking":
            rc = E.L.dfb_snapshot_write(E.h, 1, 0, fn, C.byref(ctx))
            E._ck(rc)
            stall = write = time.perf_counter() - t0
            during = []
        else:
            E.sync()
            t1 = time.perf_counter()
            f = E.snapshot_begin()
            stall = time.perf_counter() - t0
            r.update(drain_ms=round((t1 - t0) * 1e3, 2), begin_ms=round((stall - (t1 - t0)) * 1e3, 2))
            done = threading.Event()
            out = {}

            def run():
                w0 = time.perf_counter()
                try:
                    out["rc"] = E.L.dfb_frozen_write(f.f, 0, fn, C.byref(ctx))
                finally:
                    out["write"] = time.perf_counter() - w0
                    done.set()
            th = threading.Thread(target=run)
            th.start()
            during = []
            while not done.is_set():
                during.append(timed_step())
            th.join()
            assert out["rc"] == 0, E.L.dfb_frozen_error(f.f)
            f.release()
            write = out["write"] + stall
            r["write_only_s"] = round(out["write"], 3)
        after = [timed_step() for _ in range(max(0, a.window // 2 - len(during)))]
        r.update(stall_ms=round(stall * 1e3, 2), write_s=round(write, 3), steps_before=stats(before),
                 steps_during=stats(during), steps_after=stats(after))
        if during:
            r["steps_during_frac"] = round((len(during) / r["write_only_s"]) / (1e3 / statistics.mean(before)), 3)
        return r

    tmpdir = tempfile.mkdtemp()
    discard, to_fd = c_sinks(tmpdir)
    snap_bytes = st["n_keys"] * 28 + st["n_vrows"] * 64 * 8 + 40
    slots = 1 << (2 * E.table_stats()["capacity"] - 1).bit_length()        # cap = next power of 2 >= 2 x keys
    copy_bytes = 2 * (st["n_vrows"] * 128 * 4 + slots * 32)                   # read + write of rows and slots
    res["copy_gb"] = round(copy_bytes / 2 / 1e9, 2)
    res["d2d_copy_gbps"] = round(d2d_gbps(), 1)
    res["copy_ms_est"] = round(copy_bytes / 2 / (res["d2d_copy_gbps"] * 1e9) * 1e3, 1)
    for mode in ("blocking", "frozen"):
        res[f"{mode}_discard"] = window(mode, discard, -1)
    vfs = os.statvfs(tmpdir)
    if vfs.f_bavail * vfs.f_frsize > 1.2 * snap_bytes:
        for mode in ("blocking", "frozen"):
            with tempfile.TemporaryFile(dir=tmpdir) as fh:
                res[f"{mode}_file"] = window(mode, to_fd, fh.fileno())
    else:
        res["file"] = f"skipped: less than {1.2 * snap_bytes / 1e9:.1f} GB free in the temporary directory"
    for name in ("sinks.c", "sinks.so"):
        os.remove(os.path.join(tmpdir, name))
    os.rmdir(tmpdir)
    res["snapshot_gb"] = round(snap_bytes / 1e9, 2)
    res["device_name"] = torch.cuda.get_device_name(0)
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit_w"] = None
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "checkpoint_stall_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
