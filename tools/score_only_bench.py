"""What a scoring-only engine (score_only = 1, V_storage = fp32 | bf16) holds on the device and what its predict step
costs, against a training engine restored from the same snapshot.

    python tools/score_only_bench.py OUT [--windows 6] [--steps 20] [--shapes flagship,criteo39,gisette]
                                         [--train-batches N]

Per shape (those of tools/predict_bench.py) one engine is trained, its snapshot (without aux data) streamed to a
temporary file and the engine closed.  Then a training engine, an fp32 scoring engine and a bf16 scoring engine are
each created and restored from that file, and the script reports
  * device memory held after the restore: the drop of torch.cuda.mem_get_info()'s free bytes from before the engine
    was created (table, row pool and workspaces; the restore's own scratch is released), and dfb_row_bytes;
  * ms per dfb_predict_raw_dev step on the same resident batches: the three engines in alternating windows of --steps
    steps bracketed by dfb_time_mark, median and min..max over --windows windows;
  * whether the fp32 scoring engine's predictions equal the training engine's bitwise, and the largest difference of
    the bf16 engine's.
--train-batches overrides the number of training batches (the flagship's 8 make a 52 M-key model whose snapshot is
14 GB; fewer make a smaller model of the same shape, and the result says how many were used).
Writes OUT/score_only_bench.json (and prints it) with the card's name, power limit and clocks as nvidia-smi reports
them; the script sets none of them.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from difacto_b200 import capi  # noqa: E402
from predict_bench import SHAPES  # noqa: E402

ENGINES = (("training", {}), ("score_fp32", dict(score_only=1)), ("score_bf16", dict(score_only=1, V_storage="bf16")))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def labels(rows, g):
    return torch.where(torch.rand(rows, device="cuda", generator=g) < 0.3, 1.0, -1.0)


def run_shape(name, windows, steps, train_batches, tmpdir):
    make, kw, ntrain, cap = SHAPES[name]
    if train_batches:
        cap = cap // ntrain * train_batches if name != "gisette" else cap
        ntrain = train_batches
    cap = int(cap * 1.05) + 4096
    g = torch.Generator(device="cuda").manual_seed(7)
    A = capi.Engine(device=0, table_capacity=cap, **kw)
    for _ in range(ntrain):
        off, ids, val = make(g)
        rows = off.numel() - 1
        A.train_step_raw_dev(rows, ids.numel(), off, ids, val, labels(rows, g), True, True)
        A.sync()
    A.read_progress()
    st = A.table_stats()
    path = os.path.join(tmpdir, name + ".dfb")
    with open(path, "wb") as f:
        A.snapshot_to(f, save_aux=False)
    A.close()
    del off, ids, val
    torch.cuda.empty_cache()
    res = dict(train_batches=ntrain, n_keys=st["n_keys"], n_vrows=st["n_vrows"], V_dim=kw["V_dim"],
               snapshot_bytes=os.path.getsize(path))

    batches = []
    for _ in range(4):
        off, ids, val = make(g)
        rows = off.numel() - 1
        batches.append((rows, ids.numel(), off, ids, val, labels(rows, g)))
    res.update(rows=batches[0][0], nnz=batches[0][1])

    eng = {}
    for label, extra in ENGINES:
        free0 = free_bytes()
        E = capi.Engine(device=0, table_capacity=cap, V_capacity=max(st["n_vrows"], 1), **dict(kw, **extra))
        with open(path, "rb") as f:
            E.restore_from(f)
        E.sync()
        per_row, in_use = E.row_bytes()
        res[label] = dict(device_bytes_held=free0 - free_bytes(), row_bytes=per_row, row_pool_bytes_in_use=in_use)
        eng[label] = E
    os.remove(path)

    preds = {}
    for label, E in eng.items():
        out = []
        for rows, nnz, off, ids, val, lab in batches:
            p = torch.zeros(rows, device="cuda")
            E.predict_raw_dev(rows, nnz, off, ids, val, lab, p)
            E.read_progress()
            out.append(p.cpu().numpy())
        preds[label] = np.concatenate(out)
    res["score_fp32"]["bitwise_equal_to_training"] = bool(np.array_equal(preds["score_fp32"], preds["training"]))
    res["score_bf16"]["max_abs_diff_to_training"] = float(np.abs(preds["score_bf16"] - preds["training"]).max())

    def window(E):
        E.time_mark(0)
        for j in range(steps):
            rows, nnz, off, ids, val, lab = batches[j % len(batches)]
            E.predict_raw_dev(rows, nnz, off, ids, val, lab, None)
        E.time_mark(1)
        ms = E.time_elapsed_ms() / steps
        E.read_progress()
        return ms

    t = {label: [] for label in eng}
    for E in eng.values():
        window(E)
    for _ in range(windows):
        for label, E in eng.items():
            t[label].append(window(E))
    for label in eng:
        res[label]["predict_raw_dev_ms"] = dict(median=round(float(np.median(t[label])), 4),
                                                min=round(min(t[label]), 4), max=round(max(t[label]), 4))
    for E in eng.values():
        E.close()
    del batches
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--train-batches", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("score_only_bench.py measures on a GPU: none found")
    res = dict(card_power_limit_max_sm_clock_sm_clock_mem_clock=card(), lib=os.environ.get("DFB_LIB", "default"))
    with tempfile.TemporaryDirectory() as tmpdir:
        for name in args.shapes.split(","):
            res[name] = run_shape(name, args.windows, args.steps, args.train_batches, tmpdir)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "score_only_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
