"""Where the config-3 device scan spends its time, at bench.py's shape (one seeded segment tiled in HBM, one page batch).

    python tools/scan_kernel_split.py [--part both|kernels|clocks] [--rows N] [--steps K] [--clocks-lib PATH]

kernels: count / prefix / project kernel times per scan from torch.profiler (CUDA activities), in a process of its own.
clocks:  a library built with -DOBGPU_PIPE_CLOCKS (into a temporary directory, or --clocks-lib) stamps clock64 around each
         pipelined warp iteration of obgpu_count_pipe_kernel / obgpu_project_pipe_kernel (scan_small.cuh) and reports the share
         of a warp's loop spent waiting on its cp.async groups and mbarrier, issuing the next blocks' copies, and working on the
         block. The product library carries no stamps.
"both" runs the two parts in separate processes and prints one JSON line with both (the card's name, power limit and clocks
are read in the same call).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402


def build_clocks_lib(out_dir):
    """The product library's sources compiled with -DOBGPU_PIPE_CLOCKS into out_dir."""
    import __graft_entry__ as g
    b = g._build_module()
    lib = os.path.join(out_dir, "libobgpu_scan_clocks.so")
    cmd = [b.nvcc_path(), "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-DOBGPU_PIPE_CLOCKS",
           "-Xcompiler", "-fPIC", "-shared", "-o", lib] + b.SOURCES + ["-ldl"]
    r = subprocess.run(cmd, cwd=b.CSRC, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc (clocks build) failed:\n" + r.stdout + r.stderr)
    return lib


def open_cfg3(args, ob):
    """bench.py's cfg3 device setup: one seeded segment, copied `tiles` times into HBM, opened as one page batch."""
    import torch
    from oceanbase_b200.sstable import TableImage
    a = argparse.Namespace(rows=args.rows, segment_rows=args.segment_rows, rows_per_block=0, seed=args.seed)
    w, pinned, rpb, tiles, seg_rows = bench.make_cfg3_segment(a, 0, 1, pinned=True)
    seg = w.table
    stride = (seg.image.size + 127) // 128 * 128
    d_image = torch.zeros(stride * tiles + 64, dtype=torch.uint8, device="cuda")
    d_image[:seg.image.size].copy_(pinned)
    for k in range(1, tiles):
        d_image[k * stride:(k + 1) * stride].copy_(d_image[:stride])
    torch.cuda.synchronize()
    offs = (seg.offsets[None, :] + (np.arange(tiles, dtype=np.int64) * stride)[:, None]).reshape(-1)
    table = TableImage(None, offs, np.tile(seg.sizes, tiles), seg.total_rows * tiles, seg.n_cols)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)
    batch = ctx.open_batch(table, device_image_ptr=d_image.data_ptr(), host_view=False, image_size=stride * tiles)
    shape = {"rows": int(table.total_rows), "rows_per_block": int(rpb), "micro_blocks": int(table.n_blocks), "tiles": int(tiles)}
    return ctx, batch, w, int(table.total_rows * 0.13), d_image, shape


def scans(batch, w, cap, n):
    for _ in range(n):
        r = batch.scan(w.filter, w.proj, max_selected_rows=cap)
        r.info()
        r.free()


def part_kernels(args):
    import torch
    from torch.profiler import profile, ProfilerActivity
    import oceanbase_b200 as ob
    ctx, batch, w, cap, d_image, shape = open_cfg3(args, ob)
    scans(batch, w, cap, args.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        scans(batch, w, cap, args.steps)
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        if e.key.startswith("obgpu_") or "obgpu_" in e.key:
            name = e.key.split("(")[0].split("<")[0].replace("void ", "").strip()
            ms[name] = ms.get(name, 0.0) + e.device_time_total / 1e3 / args.steps
    batch.close()
    ctx.close()
    return {"shape": shape, "kernel_ms_per_scan": {k: round(v, 4) for k, v in sorted(ms.items())},
            "scan_kernels_ms": round(sum(ms.values()), 4), "steps": args.steps}


def part_clocks(args):
    import oceanbase_b200 as ob
    lib_path = args.clocks_lib or build_clocks_lib(tempfile.mkdtemp(prefix="obgpu_clocks_"))
    ob.capi.lib_path = lib_path        # the scan library is mapped on first use: before any ScanContext exists
    ctx, batch, w, cap, d_image, shape = open_cfg3(args, ob)
    get = getattr(ob.capi.lib.scan, "obgpu_pipe_clocks")
    out = (ctypes.c_ulonglong * 6)()
    scans(batch, w, cap, args.warmup)
    assert get(out) == 0
    scans(batch, w, cap, args.steps)
    assert get(out) == 0
    res = {"shape": shape, "steps": args.steps, "library": "built with -DOBGPU_PIPE_CLOCKS"}
    for k, name in enumerate(["count", "project"]):
        wait, issue, total = out[3 * k], out[3 * k + 1], out[3 * k + 2]
        if total == 0:
            res[name] = "pipelined kernel did not run"
            continue
        res[name] = {"wait_frac": round(wait / total, 4), "issue_frac": round(issue / total, 4),
                     "work_frac": round((total - wait - issue) / total, 4),
                     "cycles_per_warp_block": round(total / max(1, shape["micro_blocks"] * args.steps), 1)}
    batch.close()
    ctx.close()
    return res


def card():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except OSError:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="both", choices=["both", "kernels", "clocks"])
    ap.add_argument("--rows", type=int, default=500_000_000, help="rows of the tiled table (bench.py's cfg3 default)")
    ap.add_argument("--segment-rows", type=int, default=15_625_000)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--clocks-lib", default=None, help="a library already built with -DOBGPU_PIPE_CLOCKS")
    args = ap.parse_args()
    if args.part == "both":
        res = {"card": card()}
        for part in ("kernels", "clocks"):
            cmd = [sys.executable, os.path.abspath(__file__), "--part", part, "--rows", str(args.rows), "--segment-rows",
                   str(args.segment_rows), "--seed", str(args.seed), "--steps", str(args.steps), "--warmup", str(args.warmup)]
            if args.clocks_lib:
                cmd += ["--clocks-lib", args.clocks_lib]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                return r.returncode
            res[part] = json.loads(r.stdout.strip().splitlines()[-1])
        print(json.dumps(res))
        return 0
    import __graft_entry__ as g
    g.build()
    print(json.dumps(part_kernels(args) if args.part == "kernels" else part_clocks(args)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
