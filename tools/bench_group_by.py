"""GROUP BY over a whole cfg3-like scan: obgpu_result_group_by_values (one group per distinct value of the batch, folded on the
device) against obgpu_result_group_by (one group per (block, dictionary entry), with the per-block plan copy and every group's
aggregates sent to the host; the host merge by value that a caller would still need is not included).

The batch is cfg3's table (make_config3_like: 8 INT64 DICT + 8 VARCHAR DICT columns at the bench's block cut), scanned without a
filter and with the bench's ~10 % filter. Group columns: c0 (16 values: the low-cardinality case the fold is designed around), c3
(4 096), c6 (up to 65 536, the cap) and c8 (1 024 strings); aggregates COUNT(*), SUM / MIN / MAX of c1. Each call is timed with
CUDA events on the context's stream after a warm-up, over several repeats (median, min, max). Also printed: group counts, the
bytes each call sends to the host, and the card name and power limit read in the same run. One JSON line per case, then a summary.
obgpu_result_group_by is skipped (and says so) when its host output would exceed --old-max-gib."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import bench

GROUP_COLS = {"c0": 0, "c3": 3, "c6": 6, "c8": 8}
AGGS = [(0, -1), (1, 1), (3, 1), (4, 1)]      # COUNT(*), SUM(c1), MIN(c1), MAX(c1)
COLDESC_BYTES = 96


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def timed(fn, stream, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out = fn()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return out, {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--old-max-gib", type=float, default=8.0)
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
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    batch = ctx.open_batch(table)
    lib = ob.capi.lib
    spec = np.array(AGGS, dtype=np.int32)
    lines = []
    info = {"card": card(), "rows": table.total_rows, "blocks": table.n_blocks, "rows_per_block": rpb}
    print(json.dumps(info), flush=True)
    for fname, flt in (("none", None), ("bench 10 %", w.filter)):
        res = batch.scan(flt, [0])
        sel = res.selected_rows
        for gname, gc in GROUP_COLS.items():
            ng, kb, hn = C.c_int64(), C.c_int64(), C.c_int32()

            def new_path():
                rc = lib.obgpu_result_group_by_values(res._h, gc, spec.ctypes.data, len(AGGS), C.byref(ng), C.byref(kb), C.byref(hn))
                assert rc == 0, rc
                keys = np.empty(ng.value + 1, dtype=np.int64)
                heap = np.empty(max(kb.value, 1), dtype=np.uint8)
                out = np.empty((len(AGGS), max(ng.value, 1), 2), dtype=np.int64)
                assert lib.obgpu_result_fetch_groups(res._h, keys.ctypes.data, heap.ctypes.data, out.ctypes.data) == 0
                return ng.value

            groups, t_new = timed(new_path, stream, args.reps, args.warmup)
            new_bytes = (groups + 1) * 8 + kb.value + len(AGGS) * groups * 16 + 48
            row = {"filter": fname, "selected_rows": sel, "group_col": gname, "groups": groups, "key_bytes": kb.value,
                   "group_by_values": t_new, "group_by_values_host_bytes": new_bytes}
            # the per-(block, entry) path: its size first, then the timed call with its host output
            total = C.c_int64()
            goff = np.zeros(table.n_blocks + 1, dtype=np.int64)
            dummy = np.zeros(2 * len(AGGS), dtype=np.int64)
            rc = lib.obgpu_result_group_by(res._h, gc, spec.ctypes.data, len(AGGS), goff.ctypes.data, dummy.ctypes.data, 0, C.byref(total))
            assert rc in (0, ob.OB_BUF_NOT_ENOUGH), rc
            old_bytes = table.n_blocks * COLDESC_BYTES + len(AGGS) * total.value * 16 + 4
            row["group_by_groups"] = total.value
            row["group_by_host_bytes"] = old_bytes
            if old_bytes > args.old_max_gib * (1 << 30):
                row["group_by"] = "skipped: host output over --old-max-gib"
            else:
                host_out = np.empty(len(AGGS) * total.value * 2, dtype=np.int64)

                def old_path():
                    assert lib.obgpu_result_group_by(res._h, gc, spec.ctypes.data, len(AGGS), goff.ctypes.data, host_out.ctypes.data,
                                                     total.value, C.byref(total)) == 0
                    return total.value

                _, row["group_by"] = timed(old_path, stream, args.reps, args.warmup)
                del host_out
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
