"""What scoring-only ranks (score_only = 1, V_storage = fp32 | bf16) save in the fused sharded store.

    python tools/score_only_shard_bench.py OUT [--steps 20] [--windows 5]

Two ranks, on two GPUs when there are two, otherwise both on GPU 0.  A model is trained by two training ranks on
batches of bench.py's flagship shape (65536 rows x 100 binary ids, V_dim 64, V_threshold 0, feature counts pushed, so
every key gets a V row); the ids come from a pool of 2^pool_bits, so that the model fits the host as a snapshot
(without aux data) and the predict batches hit it.  The same snapshots are then loaded three ways -- training-layout
ranks, fp32 scoring ranks, bf16 scoring ranks -- each store with the CLI's shard capacities (max_rows 65536,
max_nnz 256 x 65536) and a row pool sized for its keys.
  * memory: per rank, the drop in free device memory across create + dfb_shard_init + restore.
  * speed: windows of --steps sharded predict steps (both ranks, predictions copied to pinned host buffers), over 4
    batches from the pool, the three stores alternating; ms per step, median and min..max over the windows.
  * check: the fp32 scoring ranks' predictions equal the training ranks' bit for bit.
Writes OUT/score_only_shard_bench.json (and prints it), with the card's name and power limit.
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
from difacto_b200.sharded import FusedShardedStore  # noqa: E402

FLAGSHIP = dict(V_dim=64, l1=0.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=0, V_init_scale=0.01, seed=1)
MAX_ROWS = 65536
MAX_NNZ = 256 * MAX_ROWS
KINDS = {"training": {}, "fp32_scoring": dict(score_only=1), "bf16_scoring": dict(score_only=1, V_storage="bf16")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().split("\n")[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def free_bytes(devices):
    out = {}
    for d in sorted(set(devices)):
        torch.cuda.synchronize(d)
        out[d] = torch.cuda.mem_get_info(d)[0]
    return out


def batch(rng, rows, nnz, pool):
    """a raw batch as pinned host tensors: (offset, ids, label)"""
    off = torch.arange(rows + 1, dtype=torch.int64) * nnz
    ids = torch.from_numpy((rng.integers(0, pool, rows * nnz, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
                           .view(np.int64))
    lab = torch.from_numpy(np.where(rng.random(rows) < 0.3, 1.0, -1.0).astype(np.float32))
    return off.pin_memory(), ids.pin_memory(), lab.pin_memory()


def step(engines, bs, outs, train=False):
    for E, (off, ids, lab), o in zip(engines, bs, outs):
        if train:
            E.shard_begin_async(len(lab), off, ids, None, lab, True, True)
        else:
            E.shard_begin_predict_async(len(lab), off, ids, None, lab, o)
    for ph in range(5):
        for E in engines:
            E.shard_phase(ph)
    return [E.wait_step() for E in engines]


def load(kind, devices, blobs, keys):
    """one store of the given kind holding the snapshots; returns (engines, device bytes per rank)"""
    free0 = free_bytes(devices)
    cap = int(keys * 1.25) + 1024
    engines = [capi.Engine(device=d, table_capacity=cap, V_capacity=cap, **FLAGSHIP, **KINDS[kind]) for d in devices]
    FusedShardedStore.connect_local(engines, MAX_ROWS, MAX_NNZ)
    for E, b in zip(engines, blobs):
        E.restore(b)
    free1 = free_bytes(devices)
    per_rank = sum(free0[d] - free1[d] for d in free0) / len(devices)
    return engines, per_rank


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--nnz", type=int, default=100)
    ap.add_argument("--pool-bits", type=int, default=22)
    ap.add_argument("--train-steps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("score_only_shard_bench: no GPU")
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    rng = np.random.default_rng(5)
    pool = 1 << args.pool_bits
    res = dict(card=card(), devices=devices, rows=args.rows, nnz_per_row=args.nnz, V_dim=FLAGSHIP["V_dim"],
               id_pool=pool, max_rows=MAX_ROWS, max_nnz=MAX_NNZ)

    # the model: training ranks, then their snapshots (no aux data: the scoring ranks would skip it anyway)
    T = [capi.Engine(device=d, table_capacity=pool, **FLAGSHIP) for d in devices]
    FusedShardedStore.connect_local(T, MAX_ROWS, MAX_NNZ)
    outs = [torch.zeros(args.rows, dtype=torch.float32).pin_memory() for _ in devices]
    for s in range(args.train_steps):
        step(T, [batch(rng, args.rows, args.nnz, pool) for _ in devices], outs, train=True)
    blobs = [E.snapshot(False) for E in T]
    keys = max(E.table_stats()["n_keys"] for E in T)
    res["model_keys"] = sum(E.table_stats()["n_keys"] for E in T)
    res["model_vrows"] = sum(E.table_stats()["n_vrows"] for E in T)
    for E in T:
        E.close()
    del T
    torch.cuda.empty_cache()

    stores, mem = {}, {}
    for kind in KINDS:
        stores[kind], mem[kind] = load(kind, devices, blobs, keys)
    res["device_bytes_per_rank"] = {k: int(v) for k, v in mem.items()}
    res["row_bytes"] = {k: stores[k][0].row_bytes()[0] for k in KINDS}
    del blobs

    pbs = [[batch(rng, args.rows, args.nnz, pool) for _ in devices] for _ in range(4)]
    pouts = {k: [torch.zeros(args.rows, dtype=torch.float32).pin_memory() for _ in devices] for k in KINDS}
    got = {}
    for k in KINDS:                                           # warm-up, and the outputs of the first batch
        for b in pbs:
            step(stores[k], b, pouts[k])
        step(stores[k], pbs[0], pouts[k])
        got[k] = [o.numpy().tobytes() for o in pouts[k]]
    res["fp32_scoring_bitwise_equal_training"] = got["fp32_scoring"] == got["training"]
    res["bf16_scoring_max_abs_diff"] = float(max(
        np.abs(np.frombuffer(a, np.float32) - np.frombuffer(b, np.float32)).max()
        for a, b in zip(got["bf16_scoring"], got["training"])))
    ms = {k: [] for k in KINDS}
    for _ in range(args.windows):
        for k in KINDS:
            t0 = time.perf_counter()
            for i in range(args.steps):
                step(stores[k], pbs[i % len(pbs)], pouts[k])     # wait_step: every rank's step has completed
            ms[k].append((time.perf_counter() - t0) * 1e3 / args.steps)
    res["predict_ms_per_step"] = {k: dict(median=round(float(np.median(v)), 3), min=round(min(v), 3),
                                          max=round(max(v), 3)) for k, v in ms.items()}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "score_only_shard_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
