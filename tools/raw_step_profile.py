"""Kernel trace of the flagship raw-id step (bench.py's default workload) with torch.profiler:

    python tools/raw_step_profile.py OUT_DIR [--steps N]

Writes one CSV per region, one line per kernel or memset (name, stream, start_us, end_us, times relative to the
region's first kernel):
  OUT_DIR/profiled.csv  dfb_profile on: the localizer shares the main stream, so every stage runs alone
  OUT_DIR/value.csv     train_step_raw_dev back to back as bench.py times it: the localizer on its own stream
and prints, per region and stream, the summed kernel time by name; for the value region also the update kernel's
mean duration and how much of the localizer stream's kernel time falls inside the update kernels' intervals.
"""
import argparse
import collections
import csv
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from difacto_b200 import capi  # noqa: E402


def trace(fn, out_dir, name):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, name + ".pt.trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"]
          if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset")]
    t0 = min(e["ts"] for e in ev)
    rows = sorted(((e["name"], int(e["args"]["stream"]), e["ts"] - t0, e["ts"] - t0 + e["dur"]) for e in ev),
                  key=lambda r: r[2])
    with open(os.path.join(out_dir, name + ".csv"), "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["name", "stream", "start_us", "end_us"])
        w.writerows((n, s, f"{a:.3f}", f"{b:.3f}") for n, s, a, b in rows)
    return rows


def summarize(rows, title, steps):
    print(f"== {title}: per-step kernel time by stream and name (us)")
    by = collections.defaultdict(float)
    for n, s, a, b in rows:
        by[(s, n[:110])] += b - a
    for (s, n), t in sorted(by.items(), key=lambda kv: (kv[0][0], -kv[1])):
        print(f"  stream {s:3d} {t / steps:9.1f}  {n}")


def overlap(rows, steps):
    upd = [(a, b, s) for n, s, a, b in rows if n.startswith("void dfb::") and "k_bwd_update" in n]
    if not upd:
        return
    main = upd[0][2]
    loc_streams = {s for n, s, a, b in rows if "k_rev_keys" in n} - {main}
    dur = np.array([b - a for a, b, _ in upd])
    print(f"== value: k_bwd_update mean {dur.mean():.1f} us (min {dur.min():.1f}, max {dur.max():.1f}, n {len(dur)})")
    if not loc_streams:
        print("  the localizer runs on the main stream")
        return
    loc = [(a, b) for n, s, a, b in rows if s in loc_streams]
    total = sum(b - a for a, b in loc)
    inside = sum(max(0.0, min(b, ub) - max(a, ua)) for a, b in loc for ua, ub, _ in upd)
    print(f"  localizer stream(s) {sorted(loc_streams)}: {total / steps:.1f} us of kernels per step, "
          f"{100.0 * inside / max(total, 1e-9):.1f} % of it inside k_bwd_update intervals")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    os.makedirs(a.out_dir, exist_ok=True)
    sys.argv = sys.argv[:1]
    args = bench.parse_args()            # the flagship defaults
    dev = torch.device("cuda", 0)
    nb = args.working_set
    host = bench.gen_raw_set(args, nb, 1, torch)
    B, N = args.batch, args.batch * args.nnz
    U0 = len(np.unique(host[0]["ids"].numpy()))
    E = capi.Engine(device=0, table_capacity=int(nb * U0 * 1.05) + 4096, V_capacity=int(nb * U0 * 1.05) + 4096,
                    id_bits=int(np.ceil(np.log2(float(args.id_space)))), overlap_auc=1, **bench.hyper(args))
    devb = [{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in h.items()} for h in host]

    def step(t, push_cnt=False):
        d = devb[t % nb]
        E.train_step_raw_dev(B, N, d["off"], d["ids"], d["val"], d["lab"], push_cnt, True)

    for p in range(2):                   # table warm-up, as in bench.py
        for t in range(nb):
            step(t, push_cnt=(p == 0))
    E.sync()

    def profiled():
        E.profile(True)
        for t in range(a.steps):
            step(t)
        E.sync()
        E.profile(False)

    def value():
        for t in range(a.steps):
            step(t)
        E.sync()

    value()                              # warm the timed path once outside the trace
    summarize(trace(profiled, a.out_dir, "profiled"), "profiled", a.steps)
    rows = trace(value, a.out_dir, "value")
    summarize(rows, "value", a.steps)
    overlap(rows, a.steps)
    E.close()


if __name__ == "__main__":
    main()
