"""What dfb_prune_rare costs, and what it frees, at the flagship fill.

    python tools/prune_rare_bench.py OUT [--rounds 3]

  * fill: 8 raw batches of 65536 rows x 100 binary ids at bench.py's flagship settings (V_dim 64, l1 = 0,
    V_threshold = 0: every counted key with w != 0 owns a V row), feature counts pushed.  Each id is, with probability
    3/4, a draw from a hot pool of 13 M ids and otherwise a fresh draw from [0, 1e9): about 25 M keys, each with a row,
    of which the fresh ones and the hot ones drawn once (about 60 %) have fea_cnt 1.  The rows are allocated batch by
    batch, so those rows are interleaved with the kept ones.
  * prune: dfb_prune_rare(max_count = 1) timed with a host clock around the call (it ends in a device synchronise).
    Bytes: the table passes of dfb_prune (the slots read twice, every occupied slot emptied, the kept entries written,
    read back and inserted; tools/prune_bench.py), the kept entries read once more to mark their rows, and the rows
    moved, read and written whole (2 * 64 floats = 512 B each).  The call does not report how many rows moved: with the
    dropped rows spread evenly over the pool, the holes below n_vkeep = n_vrows - freed are n_vkeep * freed / n_vrows,
    and that many rows move; the number is given as such an estimate.  Achieved rate as a share of the H100 SXM
    data-sheet 3.35 TB/s.  Every round after the first refills with 8 more batches of the same mix and prunes again.
  * n_vrows and the row pool's bytes in use (dfb_row_bytes) before and after each prune.
Writes OUT/prune_rare_bench.json (and prints it), with the card's name and power limit.
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
from growth_bench import FLAGSHIP, HBM_BYTES_PER_S, NB, NNZ, ROWS, card  # noqa: E402
from prune_bench import slots, step_ms  # noqa: E402

MAX_COUNT = 1.0
HOT, P_HOT = 13 << 20, 0.75


def mixed(seed, hot):
    """NB flagship-shaped batches: each id from the hot pool with probability P_HOT, else fresh from [0, 1e9)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    off = torch.arange(ROWS + 1, device="cuda", dtype=torch.int64) * NNZ
    out = []
    for _ in range(NB):
        n = ROWS * NNZ
        pick = hot[torch.randint(0, len(hot), (n,), device="cuda", generator=g)]
        new = torch.randint(0, 10 ** 9, (n,), device="cuda", generator=g, dtype=torch.int64)
        ids = torch.where(torch.rand(n, device="cuda", generator=g) < P_HOT, pick, new)
        lab = torch.where(torch.rand(ROWS, device="cuda", generator=g) < 0.3, 1.0, -1.0)
        out.append((ROWS, n, off, ids, None, lab))
    torch.cuda.synchronize()                # written before the engine's stream reads them
    return out


def prune(E):
    st = E.table_stats()
    rb, used0 = E.row_bytes()
    cap = slots(st["capacity"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n, freed = E.prune_rare(MAX_COUNT)
    s = time.perf_counter() - t0
    after = E.table_stats()
    _, used1 = E.row_bytes()
    occ, kept = st["n_keys"], st["n_keys"] - n
    nv, nvk = st["n_vrows"], st["n_vrows"] - freed
    moved_rows = int(round(nvk * freed / nv)) if nv else 0
    table_bytes = 32 * (2 * cap + occ + 3 * kept) + 32 * kept
    row_bytes_moved = 2 * rb * moved_rows
    total = table_bytes + row_bytes_moved
    return dict(keys_before=occ, keys_after=after["n_keys"], dropped=n, n_vrows_before=nv,
                n_vrows_after=after["n_vrows"], vrows_freed=freed, row_bytes=rb, bytes_in_use_before=used0,
                bytes_in_use_after=used1, slots=cap, ms=round(s * 1e3, 2), rows_moved_est=moved_rows,
                row_bytes_moved_est=row_bytes_moved, table_bytes=table_bytes, bytes_moved_est=total,
                achieved_tb_per_s=round(total / s / 1e12, 3), hbm_share=round(total / s / HBM_BYTES_PER_S, 3),
                row_move_ms_at_datasheet=round(row_bytes_moved / HBM_BYTES_PER_S * 1e3, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    res = dict(card_and_power_limit=card(), config=dict(FLAGSHIP, max_count=MAX_COUNT, rows=ROWS, nnz_per_row=NNZ,
                                                        batches=NB, hot_pool=HOT, p_hot=P_HOT))
    E = capi.Engine(device=0, table_capacity=48 << 20, V_capacity=32 << 20, **FLAGSHIP)
    g = torch.Generator(device="cuda").manual_seed(5)
    hot = torch.randint(0, 10 ** 9, (HOT,), device="cuda", generator=g, dtype=torch.int64)
    warm = mixed(99, hot)[0]
    E.train_step_raw_dev(1024, 1024 * NNZ, warm[2][:1025], warm[3][:1024 * NNZ], None, warm[5][:1024], True, True)
    E.read_progress()
    E.prune_rare(1e30)                                          # empty again: the warm-up's keys out
    res["prunes"], res["fill_ms_per_step"] = [], []
    for r in range(args.rounds):
        res["fill_ms_per_step"].append(step_ms(E, mixed(1 + r, hot), push=True))
        res["prunes"].append(prune(E))
    res["prune_ms_median"] = round(float(np.median([p["ms"] for p in res["prunes"]])), 2)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "prune_rare_bench.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
