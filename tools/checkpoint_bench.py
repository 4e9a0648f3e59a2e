"""Streamed checkpoint at bench.py's flagship shape: snapshot / restore time, bandwidth, host and device memory.

    python tools/checkpoint_bench.py [--batches 8] [--out DIR]

The table is filled the way bench.py fills it: raw minibatches of 65536 rows x 100 binary ids uniform over
[0, 1e9), V_dim 64, V_threshold 0 and l1 0 (every key gets a V row), 8 batches ~ 52 M keys.  Measured in one call:
  * snapshot (dfb_snapshot_write) into a sink that discards, and into one that hashes (crc32) and discards, in
    GB/s of snapshot bytes, next to the pinned device-to-host copy bandwidth of the same card;
  * restore (dfb_restore_read) of half that table into a second engine, fed chunk by chunk through a bounded queue
    while the first engine's snapshot is still being written (both tables fit in 80 GB);
  * peak host RSS (getrusage) and the device memory the calls take beyond the tables (cudaMemGetInfo);
  * the whole-buffer API (dfb_snapshot / dfb_restore, a host copy of the model) at 2 M keys;
  * the card's name and power limit.
Prints one JSON line (and writes it to DIR/checkpoint_bench.json with --out).  Writes nothing to disk otherwise.
"""
import argparse
import ctypes as C
import json
import os
import queue
import resource
import subprocess
import sys
import threading
import time
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from difacto_b200 import capi  # noqa: E402

ROWS, NNZ, IDS = 65536, 100, 10 ** 9
KW = dict(V_dim=64, l1=0.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=0, V_init_scale=0.01, seed=1,
          id_bits=30)


def rss_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20     # ru_maxrss is in KiB on Linux


def filled_engine(batches, seed, rows=ROWS):
    cap = int(batches * rows * NNZ * 1.05) + 4096
    E = capi.Engine(device=0, table_capacity=cap, V_capacity=cap, **KW)
    g = torch.Generator(device="cuda").manual_seed(seed)
    off = (torch.arange(rows + 1, device="cuda", dtype=torch.int64) * NNZ)
    lab = torch.where(torch.rand(rows, device="cuda", generator=g) < 0.3, 1.0, -1.0)
    for _ in range(batches):
        ids = torch.randint(0, IDS, (rows * NNZ,), device="cuda", generator=g, dtype=torch.int64)
        E.train_step_raw_dev(rows, rows * NNZ, off, ids, None, lab, True, True)
        E.sync()
    E.read_progress()
    return E


def d2h_gbps():
    n = 256 << 20
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    h = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    for _ in range(2):
        h.copy_(d, non_blocking=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        h.copy_(d, non_blocking=True)
    b.record()
    b.synchronize()
    return 10 * n / (a.elapsed_time(b) / 1e3) / 1e9


class Sink:
    """discards (and optionally crc32-hashes) what it gets; samples the free device memory during the call"""
    def __init__(self, hash_it):
        self.hash_it, self.bytes, self.crc, self.min_free = hash_it, 0, 0, None

    def write_fn(self):
        def write(_ctx, buf, n):
            if self.hash_it:
                self.crc = zlib.crc32(memoryview((C.c_char * n).from_address(buf)), self.crc)
            f = torch.cuda.mem_get_info()[0]
            self.min_free = f if self.min_free is None else min(self.min_free, f)
            self.bytes += n
            return 0
        return capi.WRITE_FN(write)


def snapshot_into(E, sink, chunk=0):
    cb = sink.write_fn()
    t = time.perf_counter()
    rc = E.L.dfb_snapshot_write(E.h, 1, chunk, cb, None)
    E._ck(rc)
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--blob-keys", type=int, default=2_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=torch.cuda.get_device_name(0))
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res["power_limit_and_max_sm_clock"] = q.stdout.strip().split("\n")[0] if q.returncode == 0 else "unknown"
    res["pinned_d2h_GBps"] = round(d2h_gbps(), 2)
    # ---- flagship snapshot ----
    free0 = torch.cuda.mem_get_info()[0]
    E = filled_engine(args.batches, 1)
    st = E.table_stats()
    res["flagship"] = dict(n_keys=st["n_keys"], n_vrows=st["n_vrows"], capacity=st["capacity"])
    free_table = torch.cuda.mem_get_info()[0]
    rss_before = rss_gb()
    snapshot_into(E, Sink(False))                      # warm-up (module loads, CUB plans)
    s1 = Sink(False)
    t1 = snapshot_into(E, s1)
    s2 = Sink(True)
    t2 = snapshot_into(E, s2)
    res["flagship"].update(
        snapshot_bytes=s1.bytes, snapshot_discard_s=round(t1, 3), snapshot_discard_GBps=round(s1.bytes / t1 / 1e9, 2),
        snapshot_crc32_s=round(t2, 3), snapshot_crc32_GBps=round(s2.bytes / t2 / 1e9, 2),
        device_workspace_GB=round((free_table - min(s1.min_free, s2.min_free)) / 1e9, 3),
        table_device_GB=round((free0 - free_table) / 1e9, 2),
        host_peak_rss_GB_before=round(rss_before, 2), host_peak_rss_GB_after=round(rss_gb(), 2))
    E.close()
    del E
    torch.cuda.empty_cache()
    # ---- restore half the working set through a bounded queue ----
    half = max(1, args.batches // 2)
    A = filled_engine(half, 2)
    stA = A.table_stats()
    B = capi.Engine(device=0, table_capacity=stA["capacity"], V_capacity=stA["v_capacity"], **KW)
    qu = queue.Queue(maxsize=4)
    err = []

    def producer():
        try:
            def write(_ctx, buf, n):
                qu.put(C.string_at(buf, n))
                return 0
            cb = capi.WRITE_FN(write)
            A._ck(A.L.dfb_snapshot_write(A.h, 1, 0, cb, None))
        except Exception as e:      # noqa: BLE001
            err.append(e)
        qu.put(None)

    class QueueSource:
        def __init__(self):
            self.pending = b""
            self.done = False

        def read(self, n):
            while not self.pending and not self.done:
                x = qu.get()
                if x is None:
                    self.done = True
                else:
                    self.pending = x
            out, self.pending = self.pending[:n], self.pending[n:]
            return out

    rss_before = rss_gb()
    th = threading.Thread(target=producer)
    t = time.perf_counter()
    th.start()
    B.restore_from(QueueSource())
    th.join()
    tr = time.perf_counter() - t
    if err:
        raise err[0]
    stB = B.table_stats()
    assert stB["n_keys"] == stA["n_keys"] and stB["n_vrows"] == stA["n_vrows"] and B.rng_state() == A.rng_state()
    nbytes = 40 + stA["n_keys"] * 28 + stA["n_vrows"] * 64 * 8
    res["restore_half"] = dict(n_keys=stA["n_keys"], n_vrows=stA["n_vrows"], bytes=nbytes,
                               snapshot_to_restore_s=round(tr, 3), GBps=round(nbytes / tr / 1e9, 2),
                               host_peak_rss_GB_before=round(rss_before, 2), host_peak_rss_GB_after=round(rss_gb(), 2))
    A.close()
    B.close()
    del A, B
    torch.cuda.empty_cache()
    # ---- the whole-buffer API at 2 M keys ----
    rows = max(1, args.blob_keys // NNZ)
    cap = int(rows * NNZ * 1.05) + 4096
    E = filled_engine(1, 3, rows)
    t = time.perf_counter()
    blob = E.snapshot()
    ts = time.perf_counter() - t
    F = capi.Engine(device=0, table_capacity=cap, V_capacity=cap, **KW)
    t = time.perf_counter()
    F.restore(blob)
    tr = time.perf_counter() - t
    res["blob_api"] = dict(n_keys=E.table_stats()["n_keys"], bytes=len(blob), snapshot_s=round(ts, 3),
                           restore_s=round(tr, 3), GBps_snapshot=round(len(blob) / ts / 1e9, 2),
                           GBps_restore=round(len(blob) / tr / 1e9, 2))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "checkpoint_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
