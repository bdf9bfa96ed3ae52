"""ORDER BY ... LIMIT k over a cfg3-like scan: obgpu_result_top_rows (rows selected and ordered on the device, only the k rows
to the host) against today's way (project the sort and output columns of every selected row to the host, then np.lexsort /
argpartition there), on a device-resident table; and obgpu_pipeline_top_rows on a host table through the pipeline.

Cases, each without a filter and with the bench's ~10 % filter, output columns c1 and c8: ORDER BY c3 DESC LIMIT 10 and LIMIT
10 000; ORDER BY c0 LIMIT 1000 (16 values: the tie-heavy key); ORDER BY c8, c1 LIMIT 100 (a string first key). Each call is timed
with CUDA events on the context's stream after a warm-up (median, min, max over --reps). Printed per case: ms of both ways, the
bytes each sends to the host, and whether both return the same rows; the card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

import bench
from bench_group_by import card, timed

CASES = [("c3 DESC LIMIT 10", [(3, 1, 0)], 10), ("c3 DESC LIMIT 10000", [(3, 1, 0)], 10_000), ("c0 LIMIT 1000", [(0, 0, 0)], 1000),
         ("c8, c1 LIMIT 100", [(8, 0, 0), (1, 0, 0)], 100)]
OUTS = [1, 8]


def host_order(res, keys, k, n_blocks):
    """today's way: every selected row's key and output columns to the host, ordered there; returns (positions, bytes)"""
    cols = sorted({c for c, _, _ in keys} | set(OUTS))
    sel = res.selected_rows
    sort_keys, nbytes = [], 0
    for c, desc, _ in reversed(keys):          # np.lexsort: the last key is the primary one
        i = cols.index(c)
        if c >= 8:
            heap, off = res.fetch_strings(i)
            nbytes += heap.size + off.size * 8
            lens = np.diff(off)
            width = int(lens.max()) if sel else 0
            mat = np.zeros((sel, max(width, 1)), dtype=np.uint8)
            rows = np.repeat(np.arange(sel), lens)
            at = np.arange(heap.size) - np.repeat(off[:-1], lens)
            mat[rows, at] = heap
            parts = [lens] + [mat[:, j] for j in range(mat.shape[1] - 1, -1, -1)]   # bytes first, then length: a proper prefix first
            sort_keys += [(-p.astype(np.int64) if desc else p) for p in parts]
        else:
            data, _, nulls = res.fetch_col(i)
            nbytes += data.nbytes + nulls.nbytes
            v = data.view(np.int64)
            sort_keys.append(-v if desc else v)
    for c in OUTS:
        i = cols.index(c)
        if c >= 8:
            heap, off = res.fetch_strings(i)
            nbytes += heap.size + off.size * 8
        else:
            data, _, nulls = res.fetch_col(i)
            nbytes += data.nbytes + nulls.nbytes
    ids = res.fetch_row_ids()
    so = res.fetch_sel_offsets()
    nbytes += ids.nbytes + so.nbytes
    blocks = np.searchsorted(so, np.arange(sel), side="right") - 1
    order = np.lexsort([ids, blocks] + sort_keys)[:k]   # position breaks ties, as the device does
    return list(zip(blocks[order].tolist(), ids[order].tolist())), nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--host-rows", type=int, default=20_000_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import oceanbase_b200 as ob
    from oceanbase_b200.pipeline import HostScanPipeline
    from oceanbase_b200.synth import make_config3_like, rows_per_block_for_target
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    rpb = rows_per_block_for_target(make_config3_like, seed=args.seed)
    info = {"card": card(), "rows": args.rows, "host_rows": args.host_rows, "rows_per_block": rpb}
    print(json.dumps(info), flush=True)
    lines = []
    stream = torch.cuda.Stream(device=torch.device("cuda", 0))
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    w, _ = bench.build_workload(args.rows, 0, args.seed, chunk_rows=1_000_000, pinned=False, maker=make_config3_like, rows_per_block=rpb,
                                align_chunks=True, n_threads=bench.host_cpus())
    batch = ctx.open_batch(w.table)
    for fname, flt in (("none", None), ("bench 10 %", w.filter)):
        res = batch.scan(flt, [0])
        for cname, keys, k in CASES:
            (pos, rows), t_new = timed(lambda: res.top_rows(keys, OUTS, k), stream, args.reps, args.warmup)
            new_bytes = len(pos) * 8 + sum(len(r[1]) + 17 for r in rows)
            cols = sorted({c for c, _, _ in keys} | set(OUTS))
            proj = batch.scan(flt, cols, want_row_ids=True)
            _, t_old = timed(lambda: host_order(proj, keys, k, w.table.n_blocks), stream, 1, 0)
            old_pos, old_bytes = host_order(proj, keys, k, w.table.n_blocks)
            proj.free()
            row = {"table": "device", "filter": fname, "case": cname, "selected_rows": res.selected_rows, "top_rows": t_new,
                   "top_rows_host_bytes": new_bytes, "project_and_sort": t_old, "project_and_sort_host_bytes": old_bytes,
                   "same_rows": old_pos == pos}
            print(json.dumps(row), flush=True)
            lines.append(row)
        res.free()
    batch.close()
    del w
    hw, _ = bench.build_workload(args.host_rows, 0, args.seed, chunk_rows=1_000_000, pinned=False, maker=make_config3_like,
                                 rows_per_block=rpb, align_chunks=True, n_threads=bench.host_cpus())
    pipe = HostScanPipeline(0)
    one = ctx.open_batch(hw.table)
    for fname, flt in (("none", None), ("bench 10 %", hw.filter)):
        res = one.scan(flt, [0])
        for cname, keys, k in CASES:
            (out, t_pipe) = timed(lambda: pipe.top_rows(hw.table, flt, keys, OUTS, k), stream, max(1, args.reps // 2), 1)
            same = out[0] == res.top_rows(keys, OUTS, k)[0]
            row = {"table": "host pipeline", "filter": fname, "case": cname, "pipeline_top_rows": t_pipe, "same_rows_as_one_batch": same}
            print(json.dumps(row), flush=True)
            lines.append(row)
        res.free()
    one.close()
    pipe.close()
    ctx.close()
    info["card_after"] = card()
    print(json.dumps(info), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for x in [info] + lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
