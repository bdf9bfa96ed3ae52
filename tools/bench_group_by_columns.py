"""GROUP BY several columns over a whole cfg3-like scan: obgpu_result_group_by_columns (one group per distinct tuple, folded on
the device) against what a caller can do without it: the same scan projecting the group and aggregate columns, fetched to the
host, then grouped there with numpy (timed separately).

The batch is cfg3's table (make_config3_like: 8 INT64 DICT + 8 VARCHAR DICT columns at the bench's block cut), scanned without a
filter and with the bench's ~10 % filter. Key sets sit on each side of each fold-path choice: (c0, c4) Q1-shaped, 17 x 17 ids
(shared accumulators); (c0, c8) and (c0, c1, c4) dense global; (c6, c0) just over 2^20 ids and (c3, c8) hashed. Aggregates:
COUNT(*), SUM / MIN / MAX of c1. Each call and its fetch are timed with CUDA events on the context's stream after a warm-up, over
several repeats (median, min, max). The path is derived from P = prod (distinct values + 1), the distinct counts read from a
one-column group_by_values per group column on the unfiltered scan. Also printed: group counts, the bytes each way sends to the
host, and the card name and power limit read in the same run. One JSON line per case."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

import bench
from bench_group_by import card, timed

KEY_SETS = {"c0,c4": [0, 4], "c0,c8": [0, 8], "c0,c1,c4": [0, 1, 4], "c6,c0": [6, 0], "c3,c8": [3, 8]}
AGGS = [(0, -1), (1, 1), (3, 1), (4, 1)]      # COUNT(*), SUM(c1), MIN(c1), MAX(c1)
SHARED_ACC_BUDGET, DENSE_GROUPS = 48 << 10, 1 << 20


def path_of(p, n_aggs):
    if p <= DENSE_GROUPS and p * (n_aggs + 1) * 16 <= SHARED_ACC_BUDGET:
        return "shared"
    return "global" if p <= DENSE_GROUPS else "hashed"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-reps", type=int, default=1, help="repeats of the projected-scan alternative")
    ap.add_argument("--host-group-max-rows", type=int, default=20_000_000, help="numpy grouping only up to this many selected rows")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import oceanbase_b200 as ob
    from oceanbase_b200.synth import make_config3_like, rows_per_block_for_target
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    rpb = rows_per_block_for_target(make_config3_like, seed=args.seed)
    w, _ = bench.build_workload(args.rows, 0, args.seed, chunk_rows=1_000_000, pinned=False, maker=make_config3_like, rows_per_block=rpb,
                                align_chunks=True, n_threads=bench.host_cpus())
    table = w.table
    stream = torch.cuda.Stream(device=torch.device("cuda", 0))
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    batch = ctx.open_batch(table)
    lib = ob.capi.lib
    spec = np.array(AGGS, dtype=np.int32)
    lines = []
    info = {"card": card(), "rows": table.total_rows, "blocks": table.n_blocks, "rows_per_block": rpb}
    print(json.dumps(info), flush=True)
    res = batch.scan(None, [0])
    distinct = {c: len([k for k in res.group_by_values(c, [(0, -1)])[0] if k is not None]) for c in sorted({c for s in KEY_SETS.values() for c in s})}
    res.free()
    for fname, flt in (("none", None), ("bench 10 %", w.filter)):
        res = batch.scan(flt, [0])
        sel = res.selected_rows
        for kname, gcols in KEY_SETS.items():
            cols = np.array(gcols, dtype=np.int32)
            ng, kb = C.c_int64(), C.c_int64()

            def new_path():
                rc = lib.obgpu_result_group_by_columns(res._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(AGGS), C.byref(ng), C.byref(kb))
                assert rc == 0, rc
                keys = np.empty((len(cols), ng.value + 1), dtype=np.int64)
                nulls = np.empty((len(cols), max(ng.value, 1)), dtype=np.uint8)
                heap = np.empty(max(kb.value, 1), dtype=np.uint8)
                out = np.empty((len(AGGS), max(ng.value, 1), 2), dtype=np.int64)
                assert lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data) == 0
                return ng.value

            groups, t_new = timed(new_path, stream, args.reps, args.warmup)
            p = int(np.prod([distinct[c] + 1 for c in gcols], dtype=object))
            row = {"filter": fname, "selected_rows": sel, "key_set": kname, "P": p, "path": path_of(p, len(AGGS)), "groups": groups,
                   "key_bytes": kb.value, "group_by_columns": t_new,
                   "group_by_columns_host_bytes": len(cols) * (groups + 1) * 8 + len(cols) * groups + kb.value + len(AGGS) * groups * 16}
            # the alternative: project the group columns and c1 for the selected rows, fetch them, group on the host
            proj = sorted(set(gcols) | {1})
            t_scan, t_host = [], []
            strs = {c for c in proj if c >= 8}          # cfg3: c8..c15 are the VARCHAR columns
            for _ in range(args.host_reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pr = batch.scan(flt, proj)
                fetched = {c: pr.fetch_strings(j) if c in strs else pr.fetch_col(j) for j, c in enumerate(proj)}
                torch.cuda.synchronize()
                t_scan.append((time.perf_counter() - t0) * 1e3)
                host_bytes = sum(int(a.nbytes) for f in fetched.values() for a in f if a is not None)
                pr.free()
                if strs & set(gcols) or sel > args.host_group_max_rows:
                    t_host.append(None)   # string keys (variable-length bytes), or more rows than --host-group-max-rows
                    continue
                t1 = time.perf_counter()
                uk, inv = np.unique(np.stack([fetched[c][0].view(np.int64) for c in gcols], axis=1), axis=0, return_inverse=True)
                inv = inv.reshape(-1)
                v = fetched[1][0].view(np.int64)
                np.bincount(inv, minlength=len(uk))
                np.bincount(inv, weights=v.astype(np.float64), minlength=len(uk))
                t_host.append((time.perf_counter() - t1) * 1e3)
                del fetched, uk, inv
            row["projected_scan_and_fetch_ms"] = round(float(np.median(t_scan)), 3)
            row["projected_host_bytes"] = host_bytes
            row["host_numpy_group_ms"] = "not measured" if None in t_host else round(float(np.median(t_host)), 3)
            print(json.dumps(row), flush=True)
            lines.append(row)
        res.free()
    batch.close()
    ctx.close()
    info["card_after"] = card()
    print(json.dumps(info), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for x in [info] + lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
