"""The raw-id predict step (dfb_predict_raw_dev) against the validation step (dfb_train_step_raw_dev, is_train=0) on
the same resident batches of one trained engine.

    python tools/predict_bench.py OUT [--windows 6] [--steps 20]

Shapes:
  * flagship: the table filled the way tools/checkpoint_bench.py fills it (8 raw batches of 65536 rows x 100 binary
    ids uniform over [0, 1e9), V_dim 64), scored on 8 fresh batches of the same shape;
  * criteo39: 65536 rows x 39 binary ids, Zipf-distributed over 2^30 (repeated keys), criteo_sgd.conf regularisation
    (l1 10, l2 10, V_l2 10, V_threshold 10), V_dim 10;
  * gisette: 6000 rows of 5000 valued ids over [0, 5000) (long rows: the one-CTA-per-row kernel), V_dim 64.
Per shape the two paths run in alternating windows of --steps steps bracketed by dfb_time_mark; the result is the
median ms per step over the windows with the min..max spread, and the per-stage times of one profiled window of each
path (dfb_profile).  Before timing, both paths' predictions are compared bitwise on every batch.
Writes OUT/predict_bench.json (and prints it), with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from difacto_b200 import capi  # noqa: E402


def flagship(g):
    rows, nnz = 65536, 100
    off = torch.arange(rows + 1, device="cuda", dtype=torch.int64) * nnz
    ids = torch.randint(0, 10 ** 9, (rows * nnz,), device="cuda", generator=g, dtype=torch.int64)
    return off, ids, None


def criteo39(g):
    rows, nnz = 65536, 39
    off = torch.arange(rows + 1, device="cuda", dtype=torch.int64) * nnz
    u = torch.rand(rows * nnz, device="cuda", generator=g, dtype=torch.float64)
    ids = (u ** -(1.0 / 0.3)).clamp(max=2.0 ** 30).to(torch.int64)        # Zipf-like: a few very hot ids
    ids = ids * 0x9E3779B1 % (1 << 30)
    return off, ids, None


def gisette(g):
    rows, nnz = 6000, 5000
    off = torch.arange(rows + 1, device="cuda", dtype=torch.int64) * nnz
    ids = torch.randint(0, 5000, (rows * nnz,), device="cuda", generator=g, dtype=torch.int64)
    val = torch.rand(rows * nnz, device="cuda", generator=g)
    return off, ids, val


SHAPES = {
    "flagship": (flagship, dict(V_dim=64, l1=0.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=0,
                                V_init_scale=0.01, seed=1, id_bits=30), 8, 65536 * 100 * 8),
    "criteo39": (criteo39, dict(V_dim=10, l1=10, l2=10, V_l2=10, V_threshold=10, lr=0.01, V_lr=0.01, seed=1,
                                id_bits=30), 8, 65536 * 39 * 8),
    "gisette": (gisette, dict(V_dim=64, l1=0.1, lr=0.01, V_lr=0.01, V_threshold=1, seed=1), 4, 1 << 16),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def run_shape(name, windows, steps):
    make, kw, ntrain, cap = SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(7)
    E = capi.Engine(device=0, table_capacity=int(cap * 1.05) + 4096, **kw)
    for _ in range(ntrain):
        off, ids, val = make(g)
        rows = off.numel() - 1
        lab = torch.where(torch.rand(rows, device="cuda", generator=g) < 0.3, 1.0, -1.0)
        E.train_step_raw_dev(rows, ids.numel(), off, ids, val, lab, True, True)
        E.sync()
    E.read_progress()
    batches = []
    for _ in range(4):
        off, ids, val = make(g)
        rows = off.numel() - 1
        lab = torch.where(torch.rand(rows, device="cuda", generator=g) < 0.3, 1.0, -1.0)
        batches.append((rows, ids.numel(), off, ids, val, lab))
    # bitwise check on every batch
    equal = True
    for rows, nnz, off, ids, val, lab in batches:
        p1 = torch.zeros(rows, device="cuda")
        E.predict_raw_dev(rows, nnz, off, ids, val, lab, p1)
        a = E.read_progress()
        b, pv = E.train_step_raw(off.cpu().numpy().view(np.uint64), ids.cpu().numpy().view(np.uint64),
                                 None if val is None else val.cpu().numpy(), lab.cpu().numpy(), False, False, True)
        equal = equal and np.array_equal(p1.cpu().numpy(), pv) and a.auc == b.auc
    res = dict(bitwise_equal=equal, rows=batches[0][0], nnz=batches[0][1])

    def window(predict):
        E.time_mark(0)
        for j in range(steps):
            rows, nnz, off, ids, val, lab = batches[j % len(batches)]
            if predict:
                E.predict_raw_dev(rows, nnz, off, ids, val, lab, None)
            else:
                E.train_step_raw_dev(rows, nnz, off, ids, val, lab, False, False)
        E.time_mark(1)
        ms = E.time_elapsed_ms() / steps
        E.read_progress()
        return ms

    window(True)
    window(False)
    t = {True: [], False: []}
    for _ in range(windows):
        for p in (True, False):
            t[p].append(window(p))
    for p, key in ((True, "predict_raw_ms"), (False, "validation_step_ms")):
        res[key] = dict(median=round(float(np.median(t[p])), 4), min=round(min(t[p]), 4), max=round(max(t[p]), 4))
    res["speedup"] = round(res["validation_step_ms"]["median"] / res["predict_raw_ms"]["median"], 3)
    for p, key in ((True, "predict_raw_stages_ms"), (False, "validation_step_stages_ms")):
        E.profile(True)
        window(p)
        st = E.profile_read()
        E.profile(False)
        res[key] = {k: round(v["ms"] / steps, 4) for k, v in st.items() if v["count"]}
    E.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    res = dict(card_and_power_limit=card(), lib=os.environ.get("DFB_LIB", "default"))
    for name in args.shapes.split(","):
        res[name] = run_shape(name, args.windows, args.steps)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "predict_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
