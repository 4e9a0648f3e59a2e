"""What growing the sharded store's ranks (shard_growth = 1) costs.

    python tools/shard_growth_bench.py OUT [--fill 2] [--steps 10] [--windows 5]

Two ranks of the fused sharded store on one GPU, each worker at bench.py's flagship per-rank shape: raw batches of
65536 rows x 100 binary ids uniform over [0, 1e9), V_dim 64, V_threshold 0 with feature counts pushed (every key gets a
V row).  --fill batches per rank bring about 6.5 M new keys each to every owner (13 M per owner after 2).
  1. fill and growth: a store whose ranks start at table_capacity = V_capacity = 2^20 and may grow up to 18 M keys and
     V rows, against a twin pre-sized to 14 M.  Per store the fill's time (every step waited for), per rank the growths
     and host waits (dfb_growth_stats), the capacities and the device memory in use.  Then one more step over the
     first batch, timed alone: its owners receive 6.5 M keys again, so the grown ranks (13 M held in about 13 M) grow
     once more, to 18 M, with a rehash into a larger slot array that the lookup waits for.
  2. steady state at a capacity boundary: a store that can grow (maxima 28 M) but holds its 13 M keys in 20 M, against
     a twin of fixed 20 M ranks: the same table and pool sizes.  Its headroom (7 M) is above what a step receives
     (6.5 M), so nothing grows, but below the worst case of a step (2 x seg_keys = 13.1 M), so every step runs the
     count kernel and its growth decision waits for the count.  Windows of --steps steps over the fill's batches,
     alternating the two stores: median ms per step with the min..max spread, growths and host waits per step, and
     the device memory each store holds afterwards.
The stores' Progress must be equal step for step while they are waited for.  Writes OUT/shard_growth_bench.json (and
prints it), with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # two ranks on one GPU: one hardware queue per stream

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from difacto_b200 import capi  # noqa: E402
from difacto_b200.sharded import FusedShardedStore  # noqa: E402

FLAGSHIP = dict(V_dim=64, l1=0.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=0, V_init_scale=0.01, seed=1,
                id_bits=30)
ROWS, NNZ, S = 65536, 100, 2
M = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def used_bytes():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def batch(rank, j):
    rng = np.random.default_rng(1000 * rank + j)
    off = (np.arange(ROWS + 1) * NNZ).astype(np.uint64)
    ids = rng.integers(0, 10 ** 9, ROWS * NNZ).astype(np.uint64)
    lab = np.where(rng.random(ROWS) < 0.3, 1.0, -1.0).astype(np.float32)
    return off, ids, None, lab


def store(ekw):
    engines = [capi.Engine(device=0, **FLAGSHIP, **ekw) for _ in range(S)]
    FusedShardedStore.connect_local(engines, max_rows=ROWS, max_nnz=ROWS * NNZ)
    return engines


def step(engines, batches, push_cnt, wait=True):
    for E, (off, ids, val, lab) in zip(engines, batches):
        E.shard_begin_async(len(lab), off, ids, val, lab, push_cnt=push_cnt, is_train=True)
    for phase in range(5):
        for E in engines:
            E.shard_phase(phase)
    if wait:
        return [tuple(E.wait_step().as_dict().values()) for E in engines]


def delta(E, g0):
    return [tuple(x - y for x, y in zip(E_.growth_stats(), g)) for E_, g in zip(E, g0)]


def fill(E, batches):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    progs = [step(E, b, True) for b in batches]
    torch.cuda.synchronize()
    return progs, dict(fill_ms=round((time.perf_counter() - t0) * 1e3, 1),
                       growths_and_host_waits=[E_.growth_stats() for E_ in E], table_stats=[E_.table_stats() for E_ in E])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--fill", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    batches = [[batch(r, j) for r in range(S)] for j in range(a.fill)]
    res = dict(card=card(), ranks_on_one_gpu=S, rows=ROWS, nnz_per_row=NNZ, fill_batches_per_rank=a.fill)
    base = used_bytes()
    res["device_bytes_free_at_start"] = torch.cuda.mem_get_info()[0]

    # 1. fill from 2^20 and one growth step
    stores, progs = {}, {}
    for name, ekw in (("grown", dict(table_capacity=M, V_capacity=M, table_capacity_max=18 * M, V_capacity_max=18 * M,
                                     shard_growth=1)),
                      ("presized", dict(table_capacity=14 * M, V_capacity=14 * M))):
        m0 = used_bytes()
        stores[name] = store(ekw)
        progs[name], r = fill(stores[name], batches)
        r["device_bytes"] = used_bytes() - m0
        res[name] = r
    assert progs["grown"] == progs["presized"], "the grown store's Progress differs from the pre-sized one's"
    for name, E in stores.items():
        g0 = [E_.growth_stats() for E_ in E]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        progs[name] = step(E, batches[0], False)
        res[name]["growth_step_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        res[name]["growth_step_growths_and_host_waits"] = delta(E, g0)
        res[name]["capacities_after_growth_step"] = [E_.table_stats() for E_ in E]
    assert progs["grown"] == progs["presized"], "the growth step's Progress differs"
    for E in stores.values():
        for E_ in E:
            E_.close()
    stores = {}
    torch.cuda.synchronize()

    # 2. steady state at a capacity boundary
    for name, ekw in (("boundary", dict(table_capacity=20 * M, V_capacity=20 * M, table_capacity_max=28 * M,
                                        V_capacity_max=28 * M, shard_growth=1)),
                      ("fixed", dict(table_capacity=20 * M, V_capacity=20 * M))):
        m0 = used_bytes()
        stores[name] = store(ekw)
        progs[name], r = fill(stores[name], batches)
        r["device_bytes_after_fill"] = used_bytes() - m0
        res[name] = r
    assert progs["boundary"] == progs["fixed"], "the growable store's Progress differs from the fixed one's"
    for E in stores.values():                       # warm-up, waited for
        for j in range(2 * a.fill):
            step(E, batches[j % a.fill], False)
    g0 = {name: [E_.growth_stats() for E_ in E] for name, E in stores.items()}
    times = {name: [] for name in stores}
    for w in range(a.windows):
        for name, E in stores.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(a.steps):
                step(E, batches[i % a.fill], False, wait=False)
            for E_ in E:
                E_.sync()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / a.steps)
    n = a.windows * a.steps
    for name, E in stores.items():
        t = sorted(times[name])
        res[name]["steady_ms_per_step"] = dict(median=round(t[len(t) // 2], 3), min=round(t[0], 3), max=round(t[-1], 3))
        res[name]["steady_growths_and_host_waits_per_step"] = [tuple(x / n for x in d) for d in delta(E, g0[name])]
        res[name]["table_stats_after_steady"] = [E_.table_stats() for E_ in E]
    # the fixed store does not change size; the rest of what is in use is the growable store's
    res["fixed"]["device_bytes_after_steady"] = res["fixed"]["device_bytes_after_fill"]
    res["boundary"]["device_bytes_after_steady"] = used_bytes() - base - res["fixed"]["device_bytes_after_fill"]
    res["device_bytes_before"] = base
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out, "shard_growth_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
