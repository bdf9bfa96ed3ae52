"""End-to-end host pipeline over stored (compressed) micro-blocks: obgpu_pipeline_scan from pinned host memory.

Per table and stored variant, three legs:
  plain    -- the plain image through the pipeline (what a caller that already holds decompressed blocks pays);
  stored   -- the stored image through the pipeline with compressor_type set: the device decodes every page batch;
  cpu+plain-- the stored payloads decompressed on --cpu-threads CPU threads (zlib streams through Python's zlib, which releases
              the GIL), then the plain pipeline: what a host without device decode pays. Only zlib variants have this leg.
Per leg: ms per pass, rows/s, h2d_bytes, d2h_bytes, kernel_launches. Selected rows and the aggregate must agree across legs.

Tables: the bench_decompress.py shape (key, small integer, 9-byte VARCHAR) at --rows, and a cfg3-shaped segment as the control
(its blocks barely compress, so they mostly stay raw). Prints one JSON line with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pinned_copy(table):
    import torch
    from oceanbase_b200.sstable import TableImage
    t = torch.empty(table.image.size, dtype=torch.uint8, pin_memory=True)
    img = t.numpy()
    img[:] = table.image
    out = TableImage(img, table.offsets, table.sizes, table.total_rows, table.n_cols)
    out._pin = t
    return out


def cpu_decompress_zlib(stored, threads):
    """Stored zlib blocks -> a plain image (blocks 128-byte aligned, header rewritten as plain), on `threads` threads."""
    from oceanbase_b200.sstable import TableImage
    import lz4_ref
    img = stored.image
    fields = [lz4_ref.header_fields(stored.block(i)) for i in range(stored.n_blocks)]
    dst_sizes = np.array([hs + dl for hs, dl, _ in fields], dtype=np.int64)
    dst_off = np.concatenate([[0], np.cumsum((dst_sizes + 127) // 128 * 128)[:-1]]).astype(np.int64)
    out = np.zeros(int(dst_off[-1] + dst_sizes[-1]) + 128, dtype=np.uint8)

    def one(i):
        hs, dl, zl = fields[i]
        o = int(stored.offsets[i])
        d = int(dst_off[i])
        out[d:d + hs] = img[o:o + hs]
        payload = img[o + hs:o + hs + zl]
        out[d + hs:d + hs + dl] = np.frombuffer(zlib.decompress(payload.tobytes()), dtype=np.uint8) if zl != dl else payload
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, range(stored.n_blocks)))
    return TableImage(out, dst_off, dst_sizes, stored.total_rows, stored.n_cols)


def run_leg(pipe, table, flt, proj, aggs, bpb, hint, compressor, reps, prep=None):
    import torch
    times, out = [], None
    for r in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        t = prep() if prep else table
        out = pipe.scan(t, flt, proj, blocks_per_batch=bpb, selectivity_hint=hint, aggs=aggs, no_row_output=True, compressor=compressor)
        torch.cuda.synchronize()
        if r:
            times.append((time.perf_counter() - t0) * 1e3)
    ms = float(np.median(times))
    return {"ms": ms, "rows_per_s": table.total_rows / (ms / 1e3), "h2d_bytes": out.h2d_bytes, "d2h_bytes": out.d2h_bytes,
            "kernel_launches": out.kernel_launches, "selected": out.selected_rows, "aggregates": [str(x) for x in out.aggregates]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=8_000_000)
    ap.add_argument("--rpb", type=int, default=1400)
    ap.add_argument("--cfg3-rows", type=int, default=4_000_000)
    ap.add_argument("--workers", type=int, default=3)
    ap.add_argument("--cpu-threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU measurement path")
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.pipeline import HostScanPipeline
    from oceanbase_b200.sstable import compress_table
    from oceanbase_b200.synth import make_config3_like
    import bench_decompress as bd
    name, power = bd.card()
    res = {"card": name, "power_limit_and_max_sm_clock": power, "tables": {}}
    t_dec = bd.make_table(a.rows, a.rpb)
    w3 = make_config3_like(rows=a.cfg3_rows, rows_per_block=133, seed=3)
    tables = {"decompress_shape": (t_dec, ob.White(1, ob.WHITE_OP_LT, (10,)), [0, 1], [(ob.AGG_SUM, 1, -1), (ob.AGG_COUNT, 0, -1)]),
              "cfg3_segment": (w3.table, w3.filter, [c for c, s in zip(w3.proj, w3.proj_is_string) if not s], [(ob.AGG_COUNT, 0, -1)])}
    pipe = HostScanPipeline(0, n_workers=a.workers)
    for tname, (table, flt, proj, aggs) in tables.items():
        bpb = max(1, table.n_blocks // 24)
        plain = pinned_copy(table)
        variants = {"lz4": (capi.COMPRESSOR_LZ4, compress_table(table, capi.COMPRESSOR_LZ4)),
                    "zstd_writer": (capi.COMPRESSOR_ZSTD_1_3_8, compress_table(table, capi.COMPRESSOR_ZSTD_1_3_8)),
                    "zstd_libzstd3": (capi.COMPRESSOR_ZSTD_1_3_8, bd.reframe_libzstd(table, 3)),
                    "zlib_writer": (capi.COMPRESSOR_ZLIB, compress_table(table, capi.COMPRESSOR_ZLIB))}
        from test_gpu_lz4_blocks import _reframe_with
        variants["zlib6"] = (capi.COMPRESSOR_ZLIB, _reframe_with(table, lambda p: zlib.compress(p, 6)))
        legs = {"plain": run_leg(pipe, plain, flt, proj, aggs, bpb, 0.3, 0, a.reps)}
        tab = {"blocks": table.n_blocks, "rows": table.total_rows, "plain_bytes": int(table.image.size), "variants": {}}
        for vname, (comp, st) in variants.items():
            if st is None:
                tab["variants"][vname] = "libzstd.so.1 not present"
                continue
            sp = pinned_copy(st)
            v = {"stored_bytes": int(st.image.size), "ratio": table.image.size / st.image.size}
            try:
                v["stored"] = run_leg(pipe, sp, flt, proj, aggs, bpb, 0.3, comp, a.reps)
            except capi.ObGpuError as e:
                v["stored"] = f"failed: {e}"
            v["cpu_then_plain"] = "not measured"
            if comp == capi.COMPRESSOR_ZLIB:
                try:
                    v["cpu_then_plain"] = run_leg(pipe, sp, flt, proj, aggs, bpb, 0.3, 0, a.reps,
                                                  prep=lambda st=st: pinned_copy(cpu_decompress_zlib(st, a.cpu_threads)))
                except capi.ObGpuError as e:
                    v["cpu_then_plain"] = f"failed: {e}"
            for leg in ("stored", "cpu_then_plain"):
                if isinstance(v[leg], dict):
                    assert v[leg]["selected"] == legs["plain"]["selected"] and v[leg]["aggregates"] == legs["plain"]["aggregates"], (tname, vname, leg)
            tab["variants"][vname] = v
        tab["plain"] = legs["plain"]
        res["tables"][tname] = tab
    pipe.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
