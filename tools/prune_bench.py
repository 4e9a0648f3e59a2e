"""What dfb_prune costs, and what it frees, at the flagship shape.

    python tools/prune_bench.py OUT [--rounds 3]

  * fill: epoch 0 at bench.py's flagship shape -- 8 raw batches of 65536 rows x 100 binary ids uniform over [0, 1e9),
    V_dim 64, feature counts pushed, about 51 M keys -- with the reference's defaults l1 = 1 and V_threshold = 10, under
    which almost every key keeps w = 0 and no V row; then 8 more batches of new ids (no feature counts), the traffic of
    a run that goes on over new ids: about 100 M keys in a table of 2^28 slots (table_capacity 120 M).
  * prune: dfb_prune(max_count = 10) timed on the host around the call (it ends in a device synchronise).  Bytes moved
    by its passes: the slots read twice (count, compact), every occupied slot written empty, the kept entries written to
    the workspace, read back and inserted.  The roofline of the design is one read of the slots plus two writes of the
    kept entries; both are given, with the achieved rate as a share of the H100 SXM data-sheet 3.35 TB/s.  Every round
    after the first follows 8 batches of new ids and prunes again.
  * steps: ms per training step (engine events) on 8 batches of new ids: into the full table before the first prune,
    and into the table after each prune.
Writes OUT/prune_bench.json (and prints it), with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from difacto_b200 import capi  # noqa: E402
from growth_bench import HBM_BYTES_PER_S, NB, NNZ, ROWS, batches, card  # noqa: E402

CONF = dict(V_dim=64, l1=1.0, l2=0.0, lr=0.01, V_lr=0.01, V_l2=0.01, V_threshold=10, V_init_scale=0.01, seed=1,
            id_bits=30)
MAX_COUNT = 10.0


def slots(max_keys):
    """the table's slots: next_pow2(2 max_keys)"""
    p = 1
    while p < 2 * max_keys:
        p <<= 1
    return p


def fresh(seed):
    """8 batches at the flagship shape whose ids are new to the table (almost all: 52 M draws over [0, 1e9))"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    off = torch.arange(ROWS + 1, device="cuda", dtype=torch.int64) * NNZ
    out = []
    for _ in range(NB):
        ids = torch.randint(0, 10 ** 9, (ROWS * NNZ,), device="cuda", generator=g, dtype=torch.int64)
        lab = torch.where(torch.rand(ROWS, device="cuda", generator=g) < 0.3, 1.0, -1.0)
        out.append((ROWS, ROWS * NNZ, off, ids, None, lab))
    return out


def step_ms(E, bs, push=False):
    """ms per step over the batches bs, timed with the engine's events"""
    E.time_mark(0)
    for b in bs:
        E.train_step_raw_dev(*b[:6], push, True)
    E.time_mark(1)
    ms = E.time_elapsed_ms() / len(bs)
    E.read_progress()
    return round(ms, 3)


def prune(E):
    st = E.table_stats()
    cap = slots(st["capacity"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = E.prune(MAX_COUNT)
    s = time.perf_counter() - t0
    occ, kept = st["n_keys"], st["n_keys"] - n
    moved = 32 * (2 * cap + occ + 3 * kept)
    least = 32 * (cap + 2 * kept)
    return dict(keys_before=occ, keys_after=E.table_stats()["n_keys"], dropped=n, slots=cap, ms=round(s * 1e3, 2),
                bytes_moved=moved, achieved_tb_per_s=round(moved / s / 1e12, 3),
                hbm_share=round(moved / s / HBM_BYTES_PER_S, 3), roofline_bytes=least,
                roofline_ms=round(least / HBM_BYTES_PER_S * 1e3, 2),
                roofline_share=round(least / HBM_BYTES_PER_S / s, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    res = dict(card_and_power_limit=card(), config=dict(CONF, max_count=MAX_COUNT, rows=ROWS, nnz_per_row=NNZ,
                                                        batches=NB))
    E = capi.Engine(device=0, table_capacity=120 << 20, V_capacity=1 << 20, **CONF)
    warm = fresh(99)[0]
    E.train_step_raw_dev(1024, 1024 * NNZ, warm[2][:1025], warm[3][:1024 * NNZ], None, warm[5][:1024], False, True)
    E.read_progress()
    res["fill_ms_per_step"] = step_ms(E, batches(), push=True)     # epoch 0: feature counts pushed
    res["filled_n_keys"] = E.table_stats()["n_keys"]
    res["step_ms_into_full_table"] = step_ms(E, fresh(1))           # 8 steps of new ids on top: 51 M -> 102 M keys
    res["n_keys_before_prune"] = E.table_stats()["n_keys"]
    res["prunes"], res["step_ms_into_pruned_table"] = [], []
    for r in range(args.rounds):
        res["prunes"].append(prune(E))
        res["step_ms_into_pruned_table"].append(step_ms(E, fresh(2 + r)))   # the same traffic after the prune
    res["prune_ms_median"] = round(float(np.median([p["ms"] for p in res["prunes"]])), 2)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "prune_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
