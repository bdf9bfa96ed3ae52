"""Cost of opening LZ4-compressed (default), zstd-compressed (--compressor zstd) or zlib-compressed (--compressor zlib) micro-blocks on the device vs opening the
plain image of the same table.

Table: seeded RAW int64 key + RAW small ints + RAW 9-byte strings, ~1 GB plain (the writer's LZ4 stores it ~1.5x smaller).
Measured with CUDA events on the ctx stream (median of --reps after one warm-up), for
  host   : image in pinned host memory -> obgpu_batch_open (plain) vs obgpu_batch_open_compressed (stored form)
  device : image already in HBM        -> same two opens (plain opened without a host view: headers surveyed on the device)
  kernel : obgpu_lz4_decompress over the compressed payloads alone (decoded GB/s from the block sizes; no checksum)
and the H2D bytes of each host open. The question: opening from host memory, do the H2D bytes saved pay for the decode?

--compressor zstd (compressor 6, zstd_1.3.8; default --rows 8M): the same opens for blocks from the writer's zstd compressor
and from libzstd at levels 1 and 3 (libzstd.so.1 through ctypes), obgpu_zstd_decompress alone on each, the ratios, and a
CPU baseline: libzstd's ZSTD_decompressDCtx over the same payloads on --cpu-threads threads (one call per micro-block, what
the reference does), timed with a host clock.

--compressor zlib (compressor 4, zlib_1.0; default --rows 8M): the same for blocks from the writer's zlib compressor (fixed
Huffman) and from the system zlib at levels 1 and 6 (Python's zlib module), obgpu_zlib_decompress alone on each, and a CPU
baseline: libz.so.1's uncompress over the same payloads on --cpu-threads threads, timed with a host clock.

  python tools/bench_decompress.py [--compressor lz4|zstd|zlib] [--rows N] [--reps R] [--cpu-threads T] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"unavailable ({e})"
    return name, q


def make_table(rows, rpb, seed=1):
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, encode_table
    rng = np.random.default_rng(seed)
    key = np.arange(rows, dtype=np.int64) * 2 + 1
    small = rng.integers(0, 40, size=rows, dtype=np.int64)
    ids = rng.integers(0, 5000, size=rows)
    digits = np.stack([(ids // 10 ** k) % 10 for k in (3, 2, 1, 0)], axis=1).astype(np.uint8) + ord("0")
    heap = np.empty((rows, 9), dtype=np.uint8)
    heap[:, :5] = np.frombuffer(b"name-", dtype=np.uint8)
    heap[:, 5:] = digits
    strs = Column(capi.OBJ_VARCHAR, capi.ENC_RAW, str_heap=np.concatenate([heap.reshape(-1), [0]]).astype(np.uint8),
                  str_off=np.arange(rows + 1, dtype=np.int64) * 9)
    return encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, key), Column(capi.OBJ_INT, capi.ENC_RAW, small), strs], rpb, rowkey_cnt=1)


def timed(fn, reps):
    import torch
    s = torch.cuda.current_stream()
    out = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        obj = fn()
        e1.record(s)
        e1.synchronize()
        obj.close()
        if r:
            out.append(e0.elapsed_time(e1))
    return float(np.median(out))


def stored_sizes(stored):
    zl = stored.image.view(np.uint8)
    zlen = np.array([int(zl[o + 44:o + 48].view(np.int32)[0]) for o in stored.offsets], dtype=np.int64)
    dlen = np.array([int(zl[o + 40:o + 44].view(np.int32)[0]) for o in stored.offsets], dtype=np.int64)
    return zlen, dlen


def reframe_libzstd(table, level):
    """The table's blocks with payloads compressed by libzstd at `level` (kept raw when not smaller), checksums fixed."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_zstd_golden as golden
    from test_gpu_lz4_blocks import _reframe_with
    z = golden.libzstd()
    if z is None:
        return None
    zs = golden.Zstd(z)
    return _reframe_with(table, lambda p: zs.compress(p, level))


def stored_opens(a, compressor, variants, entry, key, cpu_decode, cpu_key):
    """For the plain table a.table: the plain opens, then per stored variant (name -> TableImage, or None when its library is missing): the host and device
    opens with `compressor`, the device entry point `entry` (obgpu_*_decompress) over the compressed payloads alone (results
    under `key`_decompress_ms / `key`_decoded_gbps), and the CPU baseline: cpu_decode() -> fn(dst, dst_len, src, src_len)
    returning the decoded length, one call per payload on --cpu-threads threads (results under `cpu_key`_ms / _decoded_gbps;
    cpu_decode None: not measured)."""
    import concurrent.futures as cf
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.capi import lib
    table = a.table
    ctx = ob.ScanContext(0, stream=torch.cuda.current_stream().cuda_stream)
    pinned_plain = torch.from_numpy(table.image).pin_memory()
    plain_h = type(table)(pinned_plain.numpy(), table.offsets, table.sizes, table.total_rows, table.n_cols)
    dev_plain = pinned_plain.cuda()
    torch.cuda.synchronize()
    res = {"open_host_plain_ms": timed(lambda: ob.PageBatch(ctx, plain_h), a.reps),
           "open_device_plain_ms": timed(lambda: ob.PageBatch(ctx, table, device_image_ptr=dev_plain.data_ptr(), host_view=False,
                                                              image_size=table.image.size), a.reps)}
    for name, stored in variants.items():
        if stored is None:
            res[name] = "not measured (library not present)"
            continue
        pinned = torch.from_numpy(stored.image).pin_memory()
        st_h = type(stored)(pinned.numpy(), stored.offsets, stored.sizes, stored.total_rows, stored.n_cols)
        dev = pinned.cuda()
        torch.cuda.synchronize()
        r = {"open_host_ms": timed(lambda: ob.PageBatch(ctx, st_h, compressor=compressor), a.reps),
             "open_device_ms": timed(lambda: ob.PageBatch(ctx, stored, device_image_ptr=dev.data_ptr(), image_size=stored.image.size,
                                                          compressor=compressor), a.reps)}
        zlen, dlen = stored_sizes(stored)
        comp = zlen < dlen
        idx = np.nonzero(comp)[0]
        in_off = (stored.offsets[idx] + 64).astype(np.int64)
        in_len = zlen[idx].astype(np.int64)
        out_len = dlen[idx].astype(np.int64)
        out_off = np.concatenate([[0], np.cumsum(out_len)[:-1]]).astype(np.int64)
        d_out = torch.empty(int(out_len.sum()), dtype=torch.uint8, device="cuda")
        stv = np.zeros(len(idx), dtype=np.int32)
        ks = []
        for rep in range(a.reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            code = getattr(lib, entry)(ctx._h, C.c_void_p(dev.data_ptr()), in_off.ctypes.data, in_len.ctypes.data,
                                       C.c_void_p(d_out.data_ptr()), out_off.ctypes.data, out_len.ctypes.data, len(idx), stv.ctypes.data)
            e1.record()
            e1.synchronize()
            assert code == 0 and (stv == 0).all()
            if rep:
                ks.append(e0.elapsed_time(e1))
        r[key + "_decompress_ms"] = float(np.median(ks))
        r[key + "_decoded_gbps"] = float(out_len.sum()) / (r[key + "_decompress_ms"] * 1e-3) / 1e9
        r.update({"compressed_blocks": int(comp.sum()), "stored_bytes": int(stored.image.size),
                  "ratio": float(table.image.size) / float(stored.image.size),
                  "payload_ratio": float(out_len.sum()) / float(max(in_len.sum(), 1))})
        if cpu_decode is None:
            r[cpu_key] = "not measured (library not present)"
        else:   # one call per compressed payload, --cpu-threads threads (ctypes drops the GIL)
            img = stored.image
            chunks = np.array_split(np.arange(len(idx)), a.cpu_threads)
            outbuf = np.empty(int(out_len.sum()), dtype=np.uint8)

            def work(ks_):
                fn = cpu_decode()
                base = img.ctypes.data
                for k in ks_:
                    n = fn(C.c_void_p(outbuf.ctypes.data + int(out_off[k])), int(out_len[k]),
                           C.cast(C.c_void_p(base + int(in_off[k])), C.c_char_p), int(in_len[k]))
                    assert n == out_len[k]
                return len(ks_)
            with cf.ThreadPoolExecutor(a.cpu_threads) as ex:
                list(ex.map(work, chunks))   # warm-up
                cpu = []
                for _ in range(a.reps):
                    t1 = time.perf_counter()
                    list(ex.map(work, chunks))
                    cpu.append((time.perf_counter() - t1) * 1e3)
            r[cpu_key + "_ms"] = float(np.median(cpu))
            r[cpu_key + "_decoded_gbps"] = float(out_len.sum()) / (r[cpu_key + "_ms"] * 1e-3) / 1e9
            r["cpu_threads"] = a.cpu_threads
        res[name] = r
        del dev, pinned
    name, power = card()
    res.update({"card": name, "power_limit_and_max_sm_clock": power, "rows_per_block": a.rpb, "n_blocks": int(table.n_blocks),
                "plain_bytes": int(table.image.size), "reps": a.reps})
    ctx.close()
    return res


def zstd_main(a):
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import compress_table
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_zstd_golden as golden
    rows = a.rows or 8_000_000
    t0 = time.time()
    a.table = make_table(rows, a.rpb)
    variants = {"writer": compress_table(a.table, capi.COMPRESSOR_ZSTD_1_3_8), "libzstd1": reframe_libzstd(a.table, 1),
                "libzstd3": reframe_libzstd(a.table, 3)}
    build_s = time.time() - t0
    z = golden.libzstd()

    def cpu_decode():   # ZSTD_decompressDCtx, one DCtx per thread
        d = z.ZSTD_createDCtx()
        return lambda dst, n, src, sn: z.ZSTD_decompressDCtx(d, dst, n, src, sn)
    res = stored_opens(a, capi.COMPRESSOR_ZSTD_1_3_8, variants, "obgpu_zstd_decompress", "zstd", cpu_decode if z else None, "cpu_libzstd")
    res.update({"compressor": "zstd_1.3.8", "rows": rows, "table_build_s": build_s,
                "libzstd": z.ZSTD_versionString().decode() if z is not None else "not present"})
    return res


def zlib_main(a):
    import zlib
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import compress_table
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_zlib_golden as golden
    from test_gpu_lz4_blocks import _reframe_with
    rows = a.rows or 8_000_000
    t0 = time.time()
    a.table = make_table(rows, a.rpb)
    variants = {"writer": compress_table(a.table, capi.COMPRESSOR_ZLIB),
                "zlib1": _reframe_with(a.table, lambda p: zlib.compress(p, 1)), "zlib6": _reframe_with(a.table, lambda p: zlib.compress(p, 6))}
    build_s = time.time() - t0
    z = golden.libz()

    def cpu_decode():   # libz's uncompress: the decoded length, or -1 when it does not return Z_OK
        def fn(dst, n, src, sn):
            dl = C.c_ulong(n)
            return dl.value if z.uncompress(dst, C.byref(dl), src, sn) == 0 else -1
        return fn
    res = stored_opens(a, capi.COMPRESSOR_ZLIB, variants, "obgpu_zlib_decompress", "zlib", cpu_decode if z else None, "cpu_libz")
    res.update({"compressor": "zlib_1.0", "rows": rows, "table_build_s": build_s,
                "libz": z.zlibVersion().decode() if z is not None else "not present"})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compressor", choices=["lz4", "zstd", "zlib"], default="lz4")
    ap.add_argument("--rows", type=int, default=None)
    ap.add_argument("--rpb", type=int, default=700)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.compressor in ("zstd", "zlib"):
        line = json.dumps(zstd_main(a) if a.compressor == "zstd" else zlib_main(a))
        print(line)
        if a.out:
            with open(a.out, "w") as f:
                f.write(line + "\n")
        return
    a.rows = a.rows or 76_000_000
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.capi import lib
    from oceanbase_b200.sstable import compress_table
    t0 = time.time()
    table = make_table(a.rows, a.rpb)
    stored = compress_table(table, capi.COMPRESSOR_LZ4)
    build_s = time.time() - t0
    hs = 64
    zl = stored.image.view(np.uint8)
    zlen = np.array([int(zl[o + 44:o + 48].view(np.int32)[0]) for o in stored.offsets], dtype=np.int64)
    dlen = np.array([int(zl[o + 40:o + 44].view(np.int32)[0]) for o in stored.offsets], dtype=np.int64)
    comp = zlen < dlen
    ctx = ob.ScanContext(0, stream=torch.cuda.current_stream().cuda_stream)
    pinned_plain = torch.from_numpy(table.image).pin_memory()
    pinned_stored = torch.from_numpy(stored.image).pin_memory()
    plain_h = type(table)(pinned_plain.numpy(), table.offsets, table.sizes, table.total_rows, table.n_cols)
    stored_h = type(stored)(pinned_stored.numpy(), stored.offsets, stored.sizes, stored.total_rows, stored.n_cols)
    dev_plain = pinned_plain.cuda()
    dev_stored = pinned_stored.cuda()
    torch.cuda.synchronize()
    res = {}
    res["open_host_plain_ms"] = timed(lambda: ob.PageBatch(ctx, plain_h), a.reps)
    res["open_host_lz4_ms"] = timed(lambda: ob.PageBatch(ctx, stored_h, compressor=capi.COMPRESSOR_LZ4), a.reps)
    res["open_device_plain_ms"] = timed(lambda: ob.PageBatch(ctx, table, device_image_ptr=dev_plain.data_ptr(), host_view=False,
                                                             image_size=table.image.size), a.reps)
    res["open_device_lz4_ms"] = timed(lambda: ob.PageBatch(ctx, stored, device_image_ptr=dev_stored.data_ptr(),
                                                           image_size=stored.image.size, compressor=capi.COMPRESSOR_LZ4), a.reps)
    # the decoder alone over the compressed payloads (tables in host memory, one launch)
    idx = np.nonzero(comp)[0]
    in_off = (stored.offsets[idx] + hs).astype(np.int64)
    in_len = (zlen[idx]).astype(np.int64)
    out_len = dlen[idx].astype(np.int64)
    out_off = np.concatenate([[0], np.cumsum(out_len)[:-1]]).astype(np.int64)
    d_out = torch.empty(int(out_len.sum()), dtype=torch.uint8, device="cuda")
    st = np.zeros(len(idx), dtype=np.int32)
    ks = []
    for r in range(a.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        code = lib.obgpu_lz4_decompress(ctx._h, C.c_void_p(dev_stored.data_ptr()), in_off.ctypes.data, in_len.ctypes.data,
                                        C.c_void_p(d_out.data_ptr()), out_off.ctypes.data, out_len.ctypes.data, len(idx), st.ctypes.data)
        e1.record()
        e1.synchronize()
        assert code == 0 and (st == 0).all()
        if r:
            ks.append(e0.elapsed_time(e1))
    res["lz4_decompress_ms"] = float(np.median(ks))
    res["lz4_decoded_gbps"] = float(out_len.sum()) / (res["lz4_decompress_ms"] * 1e-3) / 1e9
    name, power = card()
    res.update({
        "card": name, "power_limit_and_max_sm_clock": power, "rows": a.rows, "rows_per_block": a.rpb, "n_blocks": int(table.n_blocks),
        "compressed_blocks": int(comp.sum()), "plain_bytes": int(table.image.size), "stored_bytes": int(stored.image.size),
        "ratio": float(table.image.size) / float(stored.image.size),
        "h2d_bytes_host_plain": int(table.image.size), "h2d_bytes_host_lz4": int(stored.image.size),
        "open_host_plain_gbps": table.image.size / (res["open_host_plain_ms"] * 1e-3) / 1e9,
        "open_host_lz4_gbps_of_plain_bytes": table.image.size / (res["open_host_lz4_ms"] * 1e-3) / 1e9,
        "host_open_lz4_faster": res["open_host_lz4_ms"] < res["open_host_plain_ms"], "table_build_s": build_s, "reps": a.reps})
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
