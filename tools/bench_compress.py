"""Compressing micro-blocks on the device (obgpu_compress_blocks) against the host writer's obgpu_writer_compress_blocks over the
same plain blocks, for LZ4 (compressor 2) and zstd_1.3.8 (6). One JSON line per case, with the card and its power limit read
in the same run. Device times: CUDA events on the ctx stream, median of --reps after one warm-up. Host times: a host clock,
median of --reps, on one thread and on --cpu-threads threads over slices of the blocks (ctypes releases the GIL).
  (a) table: the tools/bench_decompress.py table (RAW int64 key, small ints, 9-byte strings), uploaded plain, then compressed
  (b) phase-B: the tools/bench_encode.py columns in HBM -> obgpu_encode_columns -> compress on the device, against
      encode -> fetch -> compress on the host
GB/s is plain input bytes over time; ratio is plain bytes over stored bytes.

  python tools/bench_compress.py [--rows N] [--enc-rows N] [--reps R] [--cpu-threads T]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def host_compress(img, off, sz, compressor, threads):
    """obgpu_writer_compress_blocks over slices of the blocks (each slice packed from offset 0, align 128)."""
    from oceanbase_b200.capi import lib
    n = len(off)
    cuts = np.linspace(0, n, threads + 1).astype(int)

    def one(k):
        a, b = cuts[k], cuts[k + 1]
        if a == b:
            return 0
        s = sz[a:b]
        out = np.empty(int(((s + 127) // 128 * 128).sum()), np.uint8)
        o_off, o_sz, used = np.zeros(b - a, np.int64), np.zeros(b - a, np.int64), C.c_int64()
        code = lib.obgpu_writer_compress_blocks(img.ctypes.data, off[a:b].ctypes.data, s.ctypes.data, int(b - a), compressor, 128,
                                                out.ctypes.data, out.size, o_off.ctypes.data, o_sz.ctypes.data, C.byref(used))
        assert code == 0, code
        return int(o_sz.sum())
    with ThreadPoolExecutor(threads) as ex:
        return sum(ex.map(one, range(threads)))


def host_ms(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def device_ms(fn, reps):
    import torch
    out = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        if r:
            out.append(e0.elapsed_time(e1))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--enc-rows", type=int, default=8_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-threads", type=int, default=16)
    a = ap.parse_args()
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction
    from bench_decompress import card, make_table
    name, power = card()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    base = {"card": name, "power_limit_and_max_sm_clock": power}

    def report(case, comp, plain, stored, dev, h1, hn, extra):
        rec = dict(base, case=case, compressor={2: "lz4", 6: "zstd_1.3.8"}[comp], plain_bytes=plain, stored_bytes=stored,
                   ratio=round(plain / stored, 3), device_ms=round(dev, 3), device_gbps=round(plain / dev / 1e6, 2),
                   host_1t_ms=round(h1, 1), host_1t_gbps=round(plain / h1 / 1e6, 3),
                   host_threads=a.cpu_threads, host_nt_ms=round(hn, 1), host_nt_gbps=round(plain / hn / 1e6, 3))
        rec.update(extra)
        print(json.dumps(rec), flush=True)

    # (a) the decompress bench's table, uploaded plain
    table = make_table(a.rows, 700)
    img = np.ascontiguousarray(table.image)
    off = np.ascontiguousarray(table.offsets, dtype=np.int64)
    sz = np.ascontiguousarray(table.sizes, dtype=np.int64)
    d_img = torch.from_numpy(img).cuda()
    d_off = torch.from_numpy(off).cuda()
    d_sz = torch.from_numpy(sz.astype(np.uint32).view(np.int32)).cuda()
    plain = int(sz.sum())
    for comp in (2, 6):
        keep = []
        dev = device_ms(lambda: keep.append(compaction.compress_blocks(ctx, d_img.data_ptr(), d_off.data_ptr(), d_sz.data_ptr(),
                                                                       table.n_blocks, comp)), a.reps)
        stored = int(keep[-1].sizes.to(torch.int64).sum())
        h1 = host_ms(lambda: host_compress(img, off, sz, comp, 1), a.reps)
        hn = host_ms(lambda: host_compress(img, off, sz, comp, a.cpu_threads), a.reps)
        assert host_compress(img, off, sz, comp, a.cpu_threads) == stored
        report("table", comp, plain, stored, dev, h1, hn, {"rows": a.rows, "rows_per_block": 700, "n_blocks": int(table.n_blocks)})
        keep.clear()
    del d_img, d_off, d_sz

    # (b) phase B: encode on the device, then compress there, against encode -> fetch -> compress on the host
    g = torch.Generator(device="cuda").manual_seed(5)
    n = a.enc_rows
    key = torch.arange(n, device="cuda", dtype=torch.int64) * 3 + 1_000_000_007
    c1 = torch.randint(0, 1 << 33, (n,), device="cuda", dtype=torch.int64, generator=g)
    c2 = torch.randint(-(1 << 62), 1 << 62, (n,), device="cuda", dtype=torch.int64, generator=g)
    c3 = torch.randint(0, 1 << 13, (n,), device="cuda", dtype=torch.int64, generator=g)
    n3 = (torch.rand((n,), device="cuda", generator=g) < 0.05).to(torch.uint8)
    cols = [(key.data_ptr(), None, capi.OBJ_INT, False), (c1.data_ptr(), None, capi.OBJ_INT, False),
            (c2.data_ptr(), None, capi.OBJ_INT, False), (c3.data_ptr(), n3.data_ptr(), capi.OBJ_INT, False)]
    enc = compaction.encode_columns(ctx, cols, n, 500, rowkey_cnt=1)
    e_img, e_off, e_sz = enc.fetch()
    enc.free()
    plain = int(e_sz.sum())
    for comp in (2, 6):
        keep = []

        def dev_path():
            e = compaction.encode_columns(ctx, cols, n, 500, rowkey_cnt=1)
            keep.append(e.compress(comp))
            e.free()
        dev = device_ms(dev_path, a.reps)
        stored = int(keep[-1].sizes.to(torch.int64).sum())
        enc_ms = device_ms(lambda: compaction.encode_columns(ctx, cols, n, 500, rowkey_cnt=1).free(), a.reps)

        def host_path(threads):
            e = compaction.encode_columns(ctx, cols, n, 500, rowkey_cnt=1)
            i, o, s = e.fetch()
            e.free()
            host_compress(i, o, s, comp, threads)
        h1 = host_ms(lambda: host_path(1), a.reps)
        hn = host_ms(lambda: host_path(a.cpu_threads), a.reps)
        report("phase-B encode+compress", comp, plain, stored, dev, h1, hn,
               {"rows": n, "rows_per_block": 500, "n_blocks": int(len(e_off)), "encode_alone_ms": round(enc_ms, 3),
                "note": "device: encode + compress (CUDA events); host: encode on the device + fetch + host compress (host clock)"})
        keep.clear()
    ctx.close()


if __name__ == "__main__":
    main()
