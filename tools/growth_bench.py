"""What capacity growth (table_capacity_max / V_capacity_max) costs.

    python tools/growth_bench.py OUT [--steps 20] [--windows 5]

  * rehash: an engine (V_dim 0) filled with 8 M (32 M) keys by dfb_dev_feacnt grows to 16 M (64 M) keys on the next
    insertion; the call that grows is timed with dfb_time_mark (the two k_table_rehash launches plus a one-key lookup).
    Bytes moved: the old table read, the new table written empty, and every entry written again; as a share of the
    H100 SXM data-sheet 3.35 TB/s.
  * fill: epoch 0 at bench.py's flagship shape -- 8 raw batches of 65536 rows x 100 binary ids uniform over [0, 1e9),
    V_dim 64, V_threshold 0 with feature counts pushed (every key gets a V row), about 51 M keys -- on an engine that starts at
    table_capacity = 2^20 and grows up to 60 M keys and V rows, against an engine pre-sized for the 8 batches.  Per
    engine: the fill's time (every step waited for), the number of growths (the capacities change at most once per
    step), the final capacities, and the most device memory in use after a step (the old table, freed in stream order
    after its rehash, is additionally held during that step).
  * steady state: after the fills, windows of --steps steps over the same 8 batches on each engine, alternating; the
    median ms per step with the min..max spread.
Writes OUT/growth_bench.json (and prints it), with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from difacto_b200 import capi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FLAGSHIP = dict(V_dim=64, l1=0.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=0, V_init_scale=0.01, seed=1,
                id_bits=30)
ROWS, NNZ, NB = 65536, 100, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def used_bytes():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def rehash(keys_from, keys_to):
    E = capi.Engine(device=0, V_dim=0, table_capacity=keys_from, table_capacity_max=keys_to)
    g = torch.Generator(device="cuda").manual_seed(3)
    chunk = keys_from // 8
    cnt = torch.ones(chunk, device="cuda")
    for _ in range(8):
        keys = torch.randint(0, 1 << 62, (chunk,), device="cuda", generator=g, dtype=torch.int64)
        E.dev_feacnt(keys, chunk, cnt)
        E.sync()
    before = E.table_stats()
    one = torch.randint(0, 1 << 62, (1,), device="cuda", generator=g, dtype=torch.int64)
    E.time_mark(0)
    E.dev_feacnt(one, 1, cnt)
    E.time_mark(1)
    ms = E.time_elapsed_ms()
    after = E.table_stats()
    old_slots, new_slots = 2 * before["capacity"], 2 * after["capacity"]    # next_pow2(2 x capacity): powers of 2 here
    moved = 32 * (old_slots + new_slots + before["n_keys"])
    E.close()
    return dict(keys=before["n_keys"], capacity=[before["capacity"], after["capacity"]], ms=round(ms, 3),
                bytes_moved=moved, hbm_share=round(moved / (ms * 1e-3) / HBM_BYTES_PER_S, 3))


def batches():
    g = torch.Generator(device="cuda").manual_seed(7)
    out = []
    off = torch.arange(ROWS + 1, device="cuda", dtype=torch.int64) * NNZ
    for _ in range(NB):
        ids = torch.randint(0, 10 ** 9, (ROWS * NNZ,), device="cuda", generator=g, dtype=torch.int64)
        lab = torch.where(torch.rand(ROWS, device="cuda", generator=g) < 0.3, 1.0, -1.0)
        out.append((ROWS, ROWS * NNZ, off, ids, None, lab))
    return out


def fill(E, bs, base):
    caps, peak = [], 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for j, (rows, nnz, off, ids, val, lab) in enumerate(bs):
        E.train_step_raw_dev(rows, nnz, off, ids, val, lab, True, True)
        st = E.table_stats()       # waits for the step
        caps.append((st["capacity"], st["v_capacity"]))
        peak = max(peak, used_bytes() - base)
    E.read_progress()
    ms = (time.perf_counter() - t0) * 1e3
    growths = sum(1 for a, b in zip(caps, caps[1:]) if a != b)
    st = E.table_stats()
    return dict(ms=round(ms, 1), growths=growths, capacity=st["capacity"], v_capacity=st["v_capacity"],
                n_keys=st["n_keys"], n_vrows=st["n_vrows"], peak_gb_after_a_step=round(peak / 2 ** 30, 2),
                capacities_after_each_step=caps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    res = dict(card_and_power_limit=card())
    res["rehash_8M_to_16M"] = rehash(8 << 20, 16 << 20)
    res["rehash_32M_to_64M"] = rehash(32 << 20, 64 << 20)
    torch.cuda.empty_cache()
    bs = batches()
    base = used_bytes()
    G = capi.Engine(device=0, table_capacity=1 << 20, table_capacity_max=60 << 20, **FLAGSHIP)
    res["fill_growing"] = fill(G, bs, base)
    base = used_bytes()
    cap = int(NB * ROWS * NNZ * 1.05) + 4096
    P = capi.Engine(device=0, table_capacity=cap, V_capacity=cap, **FLAGSHIP)
    res["fill_presized"] = fill(P, bs, base)

    def window(E):
        E.time_mark(0)
        for j in range(args.steps):
            E.train_step_raw_dev(*bs[j % NB][:6], False, True)
        E.time_mark(1)
        ms = E.time_elapsed_ms() / args.steps
        E.read_progress()
        return ms

    window(G)
    window(P)
    t = {"growing": [], "presized": []}
    for _ in range(args.windows):
        t["growing"].append(window(G))
        t["presized"].append(window(P))
    for k, v in t.items():
        res[f"steady_ms_per_step_{k}"] = dict(median=round(float(np.median(v)), 3), min=round(min(v), 3),
                                              max=round(max(v), 3))
    st = G.table_stats()
    res["growing_after_steady_state"] = dict(capacity=st["capacity"], v_capacity=st["v_capacity"])
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "growth_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
