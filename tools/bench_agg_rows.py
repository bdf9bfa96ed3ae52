"""Skip-index aggregate rows built on the device (obgpu_agg_rows) against the device encoder over the same columns
(obgpu_encode_columns_ex, RAW) and the host writer's obgpu_writer_table_agg_rows on 1 and on --cpu-cores cores. One JSON line
per case, with the card and its power limit read in the same run.
Cases: --rows rows x 1, 4 and 8 INT64 columns, with 1 % NULLs and without, rows_per_block 133 and 4096.
  size_query_ms  obgpu_agg_rows without an output buffer: reduce + size + prefix passes and the synchronisation that reads the
                 total; GB/s = rows x cols x (8 + 1 with NULLs) bytes read over it (the reduce pass reads every cell once)
  call_ms        the full call with a pinned host buffer: the passes again, the write pass and the copy of rows and offsets
  encode_ms      obgpu_encode_columns_ex over the same columns (host clock around the call and a device synchronise)
  host_*_ms      obgpu_writer_table_agg_rows over the same rows in host memory, the process pinned to 1 core, then to
                 --cpu-cores cores with that many block ranges in flight (ctypes releases the GIL)
Device and host times are medians of --reps after one warm-up. The rows are checked against the writer's once per case.

  python tools/bench_agg_rows.py [--rows N] [--reps R] [--cpu-cores C]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """(name, power limit) of GPU 0 as nvidia-smi reports them."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:   # the numbers are still printed, marked with what could not be read
        return "unknown (%s)" % type(e).__name__, "unknown"


def median_ms(fn, reps, sync=None):
    fn()
    if sync:
        sync()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        if sync:
            sync()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out)), float(min(out)), float(max(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=64 * 1024 * 1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--cpu-cores", type=int, default=16)
    a = ap.parse_args()
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction, sstable
    name, power = card()
    ctx = ob.ScanContext(0)
    n = a.rows
    all_cores = sorted(os.sched_getaffinity(0))
    rng = np.random.default_rng(11)
    host_vals = [rng.integers(-(1 << 62), 1 << 62, size=n, dtype=np.int64) for _ in range(8)]
    host_null = [(rng.random(n) < 0.01).astype(np.uint8) for _ in range(8)]
    dev_vals = [torch.from_numpy(v).cuda() for v in host_vals]
    dev_null = [torch.from_numpy(x).cuda() for x in host_null]
    sync = torch.cuda.synchronize
    for ncol in (1, 4, 8):
        for nulls in (False, True):
            for rpb in (133, 4096):
                dcols = [(dev_vals[c].data_ptr(), dev_null[c].data_ptr() if nulls else None, capi.OBJ_INT, False) for c in range(ncol)]
                arr = compaction._encode_cols(dcols)
                agg = np.arange(ncol, dtype=np.int32)
                nb = (n + rpb - 1) // rpb
                size = C.c_int64()

                def query():
                    capi.check(capi.lib.obgpu_agg_rows(ctx._h, arr, ncol, agg.ctypes.data, ncol, n, rpb, None, 0, None, C.byref(size)),
                               "obgpu_agg_rows(size)", ctx._h)
                q_ms = median_ms(query, a.reps)
                out = torch.empty(size.value, dtype=torch.uint8, pin_memory=True)
                offs = torch.empty(nb + 1, dtype=torch.int64, pin_memory=True)

                def call():
                    capi.check(capi.lib.obgpu_agg_rows(ctx._h, arr, ncol, agg.ctypes.data, ncol, n, rpb, out.data_ptr(), out.numel(),
                                                       offs.data_ptr(), C.byref(size)), "obgpu_agg_rows", ctx._h)
                c_ms = median_ms(call, a.reps)
                try:   # a RAW block of 8 columns x 4096 rows does not fit one CTA's shared memory: the encoder refuses it
                    enc_ms = median_ms(lambda: compaction.encode_columns(ctx, dcols, n, rpb).free(), a.reps, sync)
                except capi.ObGpuError as e:
                    enc_ms = None
                    enc_err = str(e)
                cols = [sstable.Column(capi.OBJ_INT, capi.ENC_RAW, host_vals[c], nulls=host_null[c] if nulls else None) for c in range(ncol)]
                want_rows, want_off = sstable.table_agg_rows(cols, list(range(ncol)), rpb)
                assert np.array_equal(offs.numpy(), want_off) and np.array_equal(out.numpy(), want_rows), "rows differ from the writer's"
                del want_rows, want_off
                inputs = sstable._inputs(cols)

                def host(parts):
                    cuts = np.linspace(0, nb, parts + 1).astype(np.int64)

                    def one(k):
                        b0, b1 = int(cuts[k]), int(cuts[k + 1])
                        if b0 == b1:
                            return
                        sub = (capi.ColInput * ncol)()
                        for c in range(ncol):   # the block range's rows: column pointers moved to its first row
                            sub[c] = inputs[c]
                            sub[c].i64 = inputs[c].i64 + b0 * rpb * 8
                            if nulls:
                                sub[c].is_null = inputs[c].is_null + b0 * rpb
                        rows = min(b1 * rpb, n) - b0 * rpb
                        sz = C.c_int64()
                        capi.check(sstable.lib.obgpu_writer_table_agg_rows(sub, ncol, agg.ctypes.data, ncol, rows, rpb, None, 0, None,
                                                                           C.byref(sz)), "obgpu_writer_table_agg_rows(size)")
                        buf = np.empty(sz.value, np.uint8)
                        off = np.empty(b1 - b0 + 1, np.int64)
                        capi.check(sstable.lib.obgpu_writer_table_agg_rows(sub, ncol, agg.ctypes.data, ncol, rows, rpb, buf.ctypes.data,
                                                                           buf.size, off.ctypes.data, C.byref(sz)), "obgpu_writer_table_agg_rows")
                    with ThreadPoolExecutor(parts) as ex:
                        list(ex.map(one, range(parts)))
                os.sched_setaffinity(0, all_cores[:1])
                h1 = median_ms(lambda: host(1), a.host_reps)
                os.sched_setaffinity(0, all_cores[:a.cpu_cores])
                hn = median_ms(lambda: host(a.cpu_cores), a.host_reps)
                os.sched_setaffinity(0, all_cores)
                read = n * ncol * (9 if nulls else 8)
                print(json.dumps({
                    "card": name, "power_limit": power, "rows": n, "cols": ncol, "nulls": "1%" if nulls else "none",
                    "rows_per_block": rpb, "n_blocks": nb, "agg_row_bytes": size.value,
                    "size_query_ms": round(q_ms[0], 3), "size_query_ms_min_max": [round(q_ms[1], 3), round(q_ms[2], 3)],
                    "reduce_gbps": round(read / q_ms[0] / 1e6, 1),
                    "call_ms": round(c_ms[0], 3), "call_ms_min_max": [round(c_ms[1], 3), round(c_ms[2], 3)],
                    "encode_ms": round(enc_ms[0], 3) if enc_ms else "not supported: " + enc_err,
                    "encode_gbps": round(read / enc_ms[0] / 1e6, 1) if enc_ms else None,
                    "host_1core_ms": round(h1[0], 1), "host_cores": min(a.cpu_cores, len(all_cores)), "host_ncore_ms": round(hn[0], 1),
                }), flush=True)
                del out, offs
    ctx.close()


if __name__ == "__main__":
    main()
