"""GROUP BY columns of any encoding (obgpu_result_group_by_any): the dictionary path on cfg3 and the cells path on cfg2 and on
columns past the dictionary fold's limits, against projecting the key and aggregate columns and grouping them with numpy.

Cases (one JSON line each, after a line with the card name and power limit read in the same run):
  cfg3   make_config3_like, --rows rows device-resident at the bench's block cut, without a filter and with the bench's ~10 %
         filter: c0, c3, c8 and (c0, c4) through group_by_any, which takes the dictionary path; the fetched bytes are checked
         against group_by_columns'. c6 and c7 together, (c6, c7), whose tuples pass the dictionary fold's hashed cap at full size,
         take the cells path there.
  cfg2   make_config2_like, --rows rows: c4 (RAW, at most 128 values), c5 (13-bit), c7 (33-bit, nearly all distinct), c0 (the
         INTEGER_BASE_DIFF key: one group per row, which folds twice) and (c4, c5), all on the cells path. Where the selection has at
         most --host-max rows, the key and aggregate columns are also projected, fetched and grouped with numpy; both must agree.
  pipe   a host table of --pipe-rows rows whose columns are OBGPU_ENC_AUTO, through HostScanPipeline.group_by_any, with how many
         page batches took the cells path.
Device calls are timed with CUDA events on the ctx's stream (median, min, max of --reps after --warmup); the pipeline and the
projection with a host clock around work that ends in a synchronise. Also printed: groups and bytes to the host."""
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

AGGS = [(0, -1), (1, 1), (3, 1), (4, 1)]      # COUNT(*), SUM(c1), MIN(c1), MAX(c1)
CFG3_KEYS = {"c0": [0], "c3": [3], "c8": [8], "c0,c4": [0, 4], "c6,c7": [6, 7]}
CFG2_AGGS = [(0, -1), (1, 6), (3, 6), (4, 6)]  # COUNT(*), SUM / MIN / MAX of c6 (a RAW column)
CFG2_KEYS = {"c4": [4], "c5": [5], "c7": [7], "c0": [0], "c4,c5": [4, 5]}


def call_any(lib, res, cols, aggs):
    c = np.array(cols, dtype=np.int32)
    spec = np.array(aggs, dtype=np.int32)
    ng, kb, path = C.c_int64(), C.c_int64(), C.c_int32()
    rc = lib.obgpu_result_group_by_any(res._h, c.ctypes.data, len(c), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb), C.byref(path))
    assert rc == 0, rc
    return fetch(lib, res, len(c), len(aggs), ng.value, kb.value) + (path.value,)


def call_columns(lib, res, cols, aggs):
    c = np.array(cols, dtype=np.int32)
    spec = np.array(aggs, dtype=np.int32)
    ng, kb = C.c_int64(), C.c_int64()
    rc = lib.obgpu_result_group_by_columns(res._h, c.ctypes.data, len(c), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb))
    return fetch(lib, res, len(c), len(aggs), ng.value, kb.value) if rc == 0 else None


def fetch(lib, res, nc, na, n, kb):
    keys = np.empty((nc, n + 1), dtype=np.int64)
    nulls = np.empty((nc, max(n, 1)), dtype=np.uint8)
    heap = np.empty(max(kb, 1), dtype=np.uint8)
    out = np.empty((na, max(n, 1), 2), dtype=np.int64)
    assert lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data) == 0
    host_bytes = keys.nbytes + nc * n + kb + na * n * 16
    return (keys, nulls[:, :n], heap[:kb], out[:, :n]), n, host_bytes


def host_group(res, cols, agg_col, n_sel):
    """the projected key and aggregate columns fetched and grouped with numpy: (groups, fetch ms, numpy ms, bytes to host)"""
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vals = [res.fetch_col(i)[0].view(np.int64)[:n_sel] for i in range(len(cols) + 1)]
    t1 = time.perf_counter()
    keys = np.stack(vals[:-1], axis=1)
    uk, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    cnt = np.bincount(inv, minlength=len(uk))
    s = np.zeros(len(uk), dtype=np.float64)
    np.add.at(s, inv, vals[-1].astype(np.float64))
    t2 = time.perf_counter()
    return len(uk), cnt, round((t1 - t0) * 1e3, 3), round((t2 - t1) * 1e3, 3), sum(v.nbytes for v in vals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--pipe-rows", type=int, default=20_000_000)
    ap.add_argument("--host-max", type=int, default=20_000_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="cfg3,cfg2,pipe")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import oceanbase_b200 as ob
    from oceanbase_b200.synth import make_config2_like, make_config3_like, rows_per_block_for_target
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    lib = ob.capi.lib
    lines = []
    info = {"card": card(), "rows": args.rows, "reps": args.reps, "warmup": args.warmup}
    print(json.dumps(info), flush=True)

    def emit(row):
        print(json.dumps(row), flush=True)
        lines.append(row)

    only = set(args.only.split(","))
    if "cfg3" in only:
        rpb = rows_per_block_for_target(make_config3_like, seed=args.seed)
        w, _ = bench.build_workload(args.rows, 0, args.seed, chunk_rows=1_000_000, pinned=False, maker=make_config3_like,
                                    rows_per_block=rpb, align_chunks=True, n_threads=bench.host_cpus())
        batch = ctx.open_batch(w.table)
        for fname, flt in (("none", None), ("bench 10 %", w.filter)):
            res = batch.scan(flt, [0])
            for kname, cols in CFG3_KEYS.items():
                (got, n, hb, path), t = timed(lambda: call_any(lib, res, cols, AGGS), stream, args.reps, args.warmup)
                same = None
                ref = call_columns(lib, res, cols, AGGS)
                if ref is not None:
                    same = all(a.tobytes() == b.tobytes() for a, b in zip(got, ref[0]))
                    assert same, (kname, fname)
                emit({"case": "cfg3", "filter": fname, "selected_rows": res.selected_rows, "key": kname, "path": path, "groups": n,
                      "group_by_any": t, "host_bytes": hb, "same_bytes_as_group_by_columns": same})
            res.free()
        batch.close()
        del w
    if "cfg2" in only:
        wl = make_config2_like(rows=args.rows, seed=args.seed, n_threads=bench.host_cpus())
        batch = ctx.open_batch(wl.table)
        for fname, flt in (("none", None), ("range 25 %", wl.filter)):
            for kname, cols in CFG2_KEYS.items():
                res = batch.scan(flt, cols + [6])
                sel = res.selected_rows
                (got, n, hb, path), t = timed(lambda: call_any(lib, res, cols, CFG2_AGGS), stream, args.reps, args.warmup)
                row = {"case": "cfg2", "filter": fname, "selected_rows": sel, "key": kname, "path": path, "groups": n, "group_by_any": t,
                       "host_bytes": hb}
                if sel <= args.host_max:
                    hg, cnt, fetch_ms, np_ms, proj_bytes = host_group(res, cols, 6, sel)
                    assert hg == n and np.array_equal(np.sort(cnt), np.sort(got[3][0, :, 0])), kname
                    row.update({"project_fetch_ms": fetch_ms, "numpy_group_ms": np_ms, "project_host_bytes": proj_bytes, "same_groups": True})
                else:
                    row["project"] = "skipped: more selected rows than --host-max"
                emit(row)
                res.free()
        batch.close()
        del wl
    if "pipe" in only:
        from oceanbase_b200.pipeline import HostScanPipeline
        from oceanbase_b200.synth import config2_columns
        from oceanbase_b200.sstable import Column, encode_table
        vals = config2_columns(args.pipe_rows, args.seed, 0)
        table = encode_table([Column(ob.capi.OBJ_INT, ob.capi.ENC_AUTO, v) for v in vals], 1400, rowkey_cnt=1, n_threads=bench.host_cpus())
        p = HostScanPipeline(0, n_workers=3)
        for kname, cols in (("c4", [4]), ("c4,c5", [4, 5]), ("c2", [2])):
            for _ in range(args.warmup):
                p.group_by_any(table, None, cols, CFG2_AGGS)
            ms = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                keys, out, stats, cells = p.group_by_any(table, None, cols, CFG2_AGGS)
                ms.append((time.perf_counter() - t0) * 1e3)
            emit({"case": "pipe", "rows": stats.total_rows, "key": kname, "groups": len(keys), "batches": stats.n_batches,
                  "cells_batches": cells, "median_ms": round(float(np.median(ms)), 3), "min_ms": round(min(ms), 3),
                  "max_ms": round(max(ms), 3)})
        p.close()
    ctx.close()
    info["card_after"] = card()
    print(json.dumps(info), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for x in [info] + lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
