"""Step time of the widths the specialised kernels do not match exactly (V_dim 0, 10, 24, 40; and 16, the width a
padded 10 runs on) on the sorted fast path against the generic kernels (force_generic=1), one GPU.

Shapes (bench.py's batch builders):
  flagship   bench.py's default: B = 65536 x 100 ids over 1e9, hyper allV (every key owns a V row)
  criteo39   the Criteo-shaped batch (39 features per row, Zipf-ish ids) with criteo_sgd.conf's regularisation
             (l1 = l2 = V_l2 = 10, V_threshold = 10)
Per (shape, V_dim) one engine of each path is warmed up on the same batches (two table passes, then W steps); then
--runs timed windows of --steps dfb_train_step_raw_dev steps each, alternating the two paths, every window measured
with dfb_time_mark (CUDA events over all of the engine's streams).  Writes <out>/vdim_bench.json and prints one
line per (shape, V_dim, path).

    python tools/vdim_bench.py OUT_DIR [--vdims 0,10,24,40,16] [--steps 20] [--warmup 3] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as benchmod  # noqa: E402

SHAPES = {"flagship": dict(workload="synthetic", hyper="allV"),
          "criteo39": dict(workload="criteo39", hyper="criteo_conf")}


def gpu_info(dev):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(dev)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:         # the numbers stay valid; the card description is then missing
        return {"error": repr(e)}


def bench_args(shape, vdim, batches):
    """bench.py's defaults (its flagship shape) for the named shape"""
    saved = sys.argv
    sys.argv = ["bench.py"]
    try:
        a = benchmod.parse_args()
    finally:
        sys.argv = saved
    a.vdim = vdim
    a.workload = SHAPES[shape]["workload"]
    a.hyper = SHAPES[shape]["hyper"]
    a.working_set = batches
    return a


def run_shape(shape, vdim, opt, torch, capi):
    args = bench_args(shape, vdim, opt.batches)
    dev = torch.device("cuda", 0)
    host = benchmod.gen_raw_set(args, opt.batches, 1, torch)
    B = host[0]["nrows"]
    devb = [dict(off=h["off"].to(dev), lab=h["lab"].to(dev), ids=h["ids"].to(dev), nnz=h["nnz"],
                 val=h["val"].to(dev) if h["val"] is not None else None) for h in host]
    probe = capi.Engine(device=0, table_capacity=1024, V_dim=vdim)
    U0 = len(probe.localize(host[0]["off"].numpy().view(np.uint64), host[0]["ids"].numpy().view(np.uint64))[1])
    probe.close()
    cap = int(opt.batches * U0 * 1.05) + 4096
    id_bits = 30 if args.workload == "synthetic" else 64          # bench.py's choice for these shapes
    kw = benchmod.hyper(args)
    engines = {p: capi.Engine(device=0, table_capacity=cap, V_capacity=cap, id_bits=id_bits, force_generic=fg, **kw)
               for p, fg in (("sorted", 0), ("generic", 1))}
    torch.cuda.synchronize()

    def step(E, b, push=False):
        d = devb[b]
        E.train_step_raw_dev(B, d["nnz"], d["off"], d["ids"], d["val"], d["lab"], push, True)

    for E in engines.values():
        for p in range(2):                                     # table warm-up: every key at its steady state
            for b in range(opt.batches):
                step(E, b, push=p == 0)
        for t in range(opt.warmup):
            step(E, t % opt.batches)
        E.sync()
        E.read_progress()
    ms = {p: [] for p in engines}
    for r in range(opt.runs):
        for p in (("sorted", "generic") if r % 2 == 0 else ("generic", "sorted")):
            E = engines[p]
            E.sync()
            E.time_mark(0)
            for t in range(opt.steps):
                step(E, t % opt.batches)
            E.time_mark(1)
            ms[p].append(E.time_elapsed_ms() / opt.steps)
            E.sync()
    out = {}
    for p, E in engines.items():
        st = E.table_stats()
        out[p] = dict(ms_per_step=ms[p], median_ms=float(np.median(ms[p])),
                      examples_per_s=float(B / (np.median(ms[p]) * 1e-3)), n_keys=st["n_keys"], n_vrows=st["n_vrows"])
        E.close()
    out["speedup_median"] = out["generic"]["median_ms"] / out["sorted"]["median_ms"]
    out.update(B=B, nnz_per_row=benchmod.nnz_of(args), unique_keys_per_batch=U0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--vdims", default="0,10,24,40,16")
    ap.add_argument("--shapes", default="flagship,criteo39")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4, help="distinct batches cycled")
    opt = ap.parse_args()
    import torch
    from difacto_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("vdim_bench: no CUDA device")
    res = dict(gpu_before=gpu_info(0), steps=opt.steps, warmup=opt.warmup, runs=opt.runs, results={})
    print(f"# {res['gpu_before']}", flush=True)
    for shape in opt.shapes.split(","):
        for vdim in [int(x) for x in opt.vdims.split(",")]:
            t0 = time.time()
            r = run_shape(shape, vdim, opt, torch, capi)
            res["results"][f"{shape}/V_dim={vdim}"] = r
            for p in ("sorted", "generic"):
                print(f"{shape:9s} V_dim={vdim:3d} {p:8s} ms/step " + " ".join(f"{x:.3f}" for x in r[p]["ms_per_step"])
                      + f"  median {r[p]['median_ms']:.3f}  {r[p]['examples_per_s'] / 1e6:.2f} M ex/s", flush=True)
            print(f"{shape:9s} V_dim={vdim:3d} generic/sorted {r['speedup_median']:.2f}x  ({time.time() - t0:.0f} s)",
                  flush=True)
    res["gpu_after"] = gpu_info(0)
    print(f"# {res['gpu_after']}", flush=True)
    os.makedirs(opt.out_dir, exist_ok=True)
    with open(os.path.join(opt.out_dir, "vdim_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
