"""GROUP BY over a host-resident cfg3 table through the scan pipeline, three ways that must return the same groups:
  entry     HostScanPipeline.group_by (obgpu_pipeline_group_by): every page batch grouped on the device, its groups merged on the
            device, only the final groups fetched;
  project   the pipeline projecting the group and aggregate columns of the selected rows to host buffers (obgpu_pipeline_scan),
            then grouped on the host with numpy, the host grouping timed apart;
  loop      the per-batch loop a caller writes without the entry: open each page batch, scan it, group_by_columns, fetch its
            groups, and merge them by value on the host with numpy (one thread, batches in order).
The table is cfg3's (make_config3_like at the bench's block cut) in pinned host memory, cut into the pipeline's default page
batches (n_blocks / 12) and run on 3 workers; no filter and the bench's ~10 % filter. Key sets are those of DESIGN §6.3: (c0, c4),
(c0, c8), (c6, c0) and (c3, c8); aggregates COUNT(*), SUM / MIN / MAX of c1. Times are host wall clock around work that ends in a
synchronise, median of --reps after --warmup, with min and max. Bytes to the host are what each way copies back. The card name and
power limit are read in the same run. The tool checks that the three ways return the same groups and aggregates. One JSON line
per case."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np

import bench
from bench_group_by import card

KEY_SETS = {"c0,c4": [0, 4], "c0,c8": [0, 8], "c6,c0": [6, 0], "c3,c8": [3, 8]}
AGGS = [(0, -1), (1, 1), (3, 1), (4, 1)]      # COUNT(*), SUM(c1), MIN(c1), MAX(c1)
STRS = set(range(8, 16))                      # cfg3: c8..c15 are the VARCHAR columns
M32, M64 = np.uint64(0xffffffff), (1 << 64) - 1


def wall(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        out = fn()
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3), "reps": reps}


def int_part(a):
    """int64 keys as big-endian bytes with the sign bit flipped: bytewise order = signed order"""
    return ((a.view(np.uint64) ^ np.uint64(1 << 63)).astype(">u8")).view(np.uint8).reshape(-1, 8)


def str_part(buf, off, lens, width):
    """strings buf[off[i]:off[i] + lens[i]] as rows of `width` bytes, zero padded (no cfg3 string holds a NUL byte)"""
    idx = off[:, None] + np.arange(width, dtype=np.int64)[None, :]
    m = np.arange(width)[None, :] < lens[:, None]
    return np.where(m, buf[np.where(m, idx, 0)], 0).astype(np.uint8)


def host_group(parts, cnt, lo, hi, mn, mx):
    """rows (key byte rows, COUNT, SUM as (lo u64, hi i64), MIN, MAX) merged by key: (unique key rows, count, lo, hi, min, max);
    the rows' 128-bit sums are added exactly in 32-bit limbs"""
    km = np.ascontiguousarray(np.concatenate(parts, axis=1))
    uk, inv = np.unique(km.view(np.dtype((np.void, km.shape[1]))).reshape(-1), return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(inv, kind="stable")
    starts = np.searchsorted(inv[order], np.arange(len(uk)))
    lo_o = lo[order]
    t0 = np.add.reduceat((lo_o & M32).astype(np.int64), starts).astype(np.uint64)
    t1 = np.add.reduceat((lo_o >> np.uint64(32)).astype(np.int64), starts).astype(np.uint64) + (t0 >> np.uint64(32))
    s_lo = (t0 & M32) | (t1 << np.uint64(32))
    s_hi = np.add.reduceat(hi[order], starts) + (t1 >> np.uint64(32)).astype(np.int64)
    return (uk, np.add.reduceat(cnt[order], starts), s_lo.view(np.int64), s_hi, np.minimum.reduceat(mn[order], starts),
            np.maximum.reduceat(mx[order], starts))


def as_tuples(uk, width_of, gcols):
    """unique key rows back to tuples of Python ints / bytes"""
    rows = np.frombuffer(uk.tobytes(), dtype=np.uint8).reshape(len(uk), -1)
    cols, at = [], 0
    for c in gcols:
        w = width_of[c]
        b = rows[:, at:at + w]
        if c in STRS:
            cols.append([bytes(r).rstrip(b"\0") for r in b])
        else:
            cols.append((np.ascontiguousarray(b).view(">u8").reshape(-1) ^ np.uint64(1 << 63)).astype(np.uint64).view(np.int64).tolist())
        at += w
    return list(zip(*cols))


def as_out(g):
    uk, cnt, lo, hi, mn, mx = g
    n = len(uk)
    out = np.zeros((4, n, 2), dtype=np.int64)
    out[0, :, 0] = cnt
    out[1, :, 0], out[1, :, 1] = lo, hi
    out[2, :, 0], out[2, :, 1] = mn, 1
    out[3, :, 0], out[3, :, 1] = mx, 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=20_000_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workers", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import oceanbase_b200 as ob
    from oceanbase_b200.pipeline import HostScanPipeline, HostOutputs, batch_bounds, split_table
    from oceanbase_b200.synth import make_config3_like, rows_per_block_for_target
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    rpb = rows_per_block_for_target(make_config3_like, seed=args.seed)
    w, _ = bench.build_workload(args.rows, 0, args.seed, chunk_rows=1_000_000, pinned=True, maker=make_config3_like, rows_per_block=rpb,
                                align_chunks=True, n_threads=bench.host_cpus())
    table = w.table
    n_blocks = table.n_blocks
    bpb = max(1, n_blocks // 12)
    pipe = HostScanPipeline(0, n_workers=args.workers)
    info = {"card": card(), "rows": table.total_rows, "blocks": n_blocks, "rows_per_block": rpb, "page_batches": len(batch_bounds(n_blocks, bpb)) - 1,
            "workers": args.workers, "pinned": True}
    print(json.dumps(info), flush=True)
    lines = []
    ctx = ob.ScanContext(0)
    parts = split_table(table, bpb)
    for fname, flt in (("none", None), ("bench 10 %", w.filter)):
        for kname, gcols in KEY_SETS.items():
            row = {"filter": fname, "key_set": kname}
            # 1. the entry
            (keys, out, stats), t = wall(lambda: pipe.group_by(table, flt, gcols, AGGS, blocks_per_batch=bpb), args.reps, args.warmup)
            n = len(keys)
            kb = sum(len(k[i]) for k in keys for i, c in enumerate(gcols) if c in STRS and k[i] is not None)
            row.update({"groups": n, "selected_rows": stats.selected_rows, "entry": t,
                        "entry_host_bytes": len(gcols) * (n + 1) * 8 + len(gcols) * n + kb + len(AGGS) * n * 16})
            # 2. the pipeline projecting the group and aggregate columns, grouped on the host
            proj = list(gcols) + [1]
            is_str = [c in STRS for c in proj]
            elem = [8] * len(proj)
            outs = HostOutputs.allocate(table.total_rows + 64 * (n_blocks // bpb + 4), is_str, elem, pinned=True)
            scan, t = wall(lambda: pipe.scan(table, flt, proj, bpb, 1.0, outputs=outs, no_row_output=False, proj_is_string=is_str,
                                             proj_elem_len=elem), args.reps, args.warmup)
            row["project"] = t
            row["project_host_bytes"] = scan.d2h_bytes
            t0 = time.perf_counter()
            cols = {c: [] for c in proj}
            for b in scan.batches:
                for j, c in enumerate(proj):
                    if c in STRS:
                        cols[c].append((b.cols[j].view(np.int64), b.lens[j].astype(np.int64)))
                    else:
                        cols[c].append(b.cols[j].view(np.int64))
            width = {c: 8 for c in proj}
            kp = []
            for c in gcols:
                if c in STRS:
                    off = np.concatenate([p for p, _ in cols[c]])
                    ln = np.concatenate([x for _, x in cols[c]])
                    width[c] = int(ln.max()) if len(ln) else 1
                    kp.append(str_part(table.image, off, ln, width[c]))
                else:
                    kp.append(int_part(np.concatenate(cols[c])))
            v = np.concatenate(cols[1])
            proj_g = host_group(kp, np.ones(len(v), dtype=np.int64), v.view(np.uint64), np.where(v < 0, -1, 0).astype(np.int64), v, v)
            row["project_host_group_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
            del scan, cols, kp, outs
            # 3. the per-batch loop with a host merge
            def loop():
                kparts, cnt, lo, hi, mn, mx = [[] for _ in gcols], [], [], [], [], []
                host = 0
                for part in parts:
                    batch = ctx.open_batch(part)
                    res = batch.scan(flt, [0])
                    k, nulls, heap, o = ob_raw(ob, res, gcols)
                    res.free()
                    batch.close()
                    m = o.shape[1]
                    host += k.nbytes + nulls.nbytes + heap.nbytes + o.nbytes
                    for i, c in enumerate(gcols):
                        if c in STRS:
                            kparts[i].append((heap, k[i, :m], k[i, 1:m + 1] - k[i, :m]))
                        else:
                            kparts[i].append(k[i, :m])
                    cnt.append(o[0, :, 0]), lo.append(o[1, :, 0].view(np.uint64)), hi.append(o[1, :, 1])
                    mn.append(o[2, :, 0]), mx.append(o[3, :, 0])
                kp = []
                for i, c in enumerate(gcols):
                    if c in STRS:
                        wd = max(int(x.max()) if len(x) else 1 for _, _, x in kparts[i])
                        width[c] = max(width.get(c, 1), wd)
                        kp.append(np.concatenate([str_part(h, off, ln, width[c]) for h, off, ln in kparts[i]]))
                    else:
                        kp.append(int_part(np.concatenate(kparts[i])))
                g = host_group(kp, *(np.concatenate(x) for x in (cnt, lo, hi, mn, mx)))
                return g, host
            (loop_g, loop_bytes), t = wall(loop, args.reps, args.warmup)
            row["loop"] = t
            row["loop_host_bytes"] = loop_bytes
            # the same groups three ways
            want_keys = as_tuples(proj_g[0], width, gcols)
            same = (keys == want_keys and np.array_equal(out, as_out(proj_g)) and as_tuples(loop_g[0], width, gcols) == want_keys
                    and np.array_equal(as_out(loop_g), out))
            row["same_groups"] = bool(same)
            print(json.dumps(row), flush=True)
            lines.append(row)
            if not same:
                raise SystemExit(f"the three ways disagree on {fname} / {kname}")
    ctx.close()
    pipe.close()
    info["card_after"] = card()
    print(json.dumps(info), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for x in [info] + lines:
                f.write(json.dumps(x) + "\n")


def ob_raw(ob, res, gcols):
    """one batch's groups as fetched: (keys, nulls, heap, out)"""
    import ctypes as C
    lib = ob.capi.lib
    cols = np.array(gcols, dtype=np.int32)
    spec = np.array(AGGS, dtype=np.int32)
    ng, kb = C.c_int64(), C.c_int64()
    rc = lib.obgpu_result_group_by_columns(res._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(AGGS), C.byref(ng), C.byref(kb))
    assert rc == 0, rc
    n = ng.value
    keys = np.empty((len(cols), n + 1), dtype=np.int64)
    nulls = np.empty((len(cols), max(n, 1)), dtype=np.uint8)
    heap = np.zeros(max(kb.value, 1) + 64, dtype=np.uint8)
    out = np.empty((len(AGGS), max(n, 1), 2), dtype=np.int64)
    assert lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data) == 0
    assert not nulls[:, :n].any(), "cfg3 group columns hold no NULL"
    return keys, nulls[:, :n], heap, out[:, :n]


if __name__ == "__main__":
    main()
