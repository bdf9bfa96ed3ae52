"""Device encoder (phase B of the compaction) alone: config-5 shaped columns (INT64 rowkey + 3 INT64 payload columns, one of
them with NULLs) already in HBM -> PAX micro-blocks + column checksums. --encoding raw writes every column RAW, auto lets every
column choose its codec per block (OBGPU_ENC_AUTO); "both" (the default) times the two arms alternately in one process. cs writes
CS_ENCODING_ROW_STORE blocks with every column CS_INTEGER, cs_auto with every column OBGPU_ENC_CS_AUTO (obgpu_encode_columns_cs_ex);
--stream-mode M[,M...] encodes their integer streams under each listed mode (obgpu_writer_set_cs_stream_encoding's meaning: 1 RAW,
0 detect, 2..6 / 8 one codec), every (encoding, mode) pair an arm of its own. Prints one JSON line per arm: ms, rows/s, image bytes, algorithmic GB/s (input columns read once + image written once) against the
H100 data-sheet HBM bandwidth, and the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    """(name, power limit) of GPU 0 as nvidia-smi reports them."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception as e:   # the numbers stay valid; say that the card could not be read
        return f"unknown ({e.__class__.__name__})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=64_000_000)
    ap.add_argument("--rows-per-block", type=int, default=500)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--encoding", default="both", choices=["raw", "auto", "both", "cs", "cs_auto"])
    ap.add_argument("--stream-mode", default="1", help="cs / cs_auto: comma-separated integer stream modes, each timed as an arm")
    ap.add_argument("--verify", action="store_true", help="also encode the rows with the host writer (at the same stream mode): "
                                                          "the images must be equal")
    a = ap.parse_args()
    modes = [int(m) for m in a.stream_mode.split(",")]
    import torch
    import bench
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = ob.ScanContext(0, stream=stream.cuda_stream)   # CUDA events below time the stream the kernels run on
    g = torch.Generator(device="cuda").manual_seed(5)
    n = a.rows
    key = torch.arange(n, device="cuda", dtype=torch.int64) * 3 + 1_000_000_007
    c1 = torch.randint(0, 1 << 33, (n,), device="cuda", dtype=torch.int64, generator=g)
    c2 = torch.randint(-(1 << 62), 1 << 62, (n,), device="cuda", dtype=torch.int64, generator=g)
    c3 = torch.randint(0, 1 << 13, (n,), device="cuda", dtype=torch.int64, generator=g)
    n3 = (torch.rand((n,), device="cuda", generator=g) < 0.05).to(torch.uint8)
    cols = [(key.data_ptr(), None, capi.OBJ_INT, False), (c1.data_ptr(), None, capi.OBJ_INT, False),
            (c2.data_ptr(), None, capi.OBJ_INT, False), (c3.data_ptr(), n3.data_ptr(), capi.OBJ_INT, False)]
    in_bytes = n * (4 * 8 + 1)
    arms = [(e, m) for e in (["raw", "auto"] if a.encoding == "both" else [a.encoding]) for m in (modes if e.startswith("cs") else [1])]
    encs = {"raw": None, "auto": [capi.ENC_AUTO] * 4, "cs": None, "cs_auto": [capi.ENC_CS_AUTO] * 4}
    writer_enc = {"raw": capi.ENC_RAW, "auto": capi.ENC_AUTO, "cs": capi.ENC_CS_INTEGER, "cs_auto": capi.ENC_CS_AUTO}
    ms = {k: [] for k in arms}
    img_bytes, nb = {}, {}
    for it in range(a.warmup + a.steps):
        for arm in arms:   # the arms alternate step by step
            kind, mode = arm
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            enc = compaction.encode_columns(ctx, cols, n, a.rows_per_block, rowkey_cnt=1, encodings=encs[kind], cs=kind.startswith("cs"),
                                            stream_mode=mode)
            e1.record()
            torch.cuda.synchronize()
            info = enc.info()
            img_bytes[arm], nb[arm] = info.image_size, info.n_blocks
            assert info.n_host_blocks == 0
            if a.verify and it == 0:
                from oceanbase_b200.sstable import Column, encode_table
                img = enc.fetch()[0]
                e = writer_enc[kind]
                host = [Column(capi.OBJ_INT, e, t.cpu().numpy()) for t in (key, c1, c2)]
                host.append(Column(capi.OBJ_INT, e, c3.cpu().numpy(), nulls=n3.cpu().numpy()))
                assert capi.lib.obgpu_writer_set_cs_stream_encoding(mode) == 0
                want = np.asarray(encode_table(host, a.rows_per_block, rowkey_cnt=1, align=128).image)
                capi.lib.obgpu_writer_set_cs_stream_encoding(1)
                assert np.array_equal(img, want), f"{arm}: the device image differs from the host writer's"
            enc.free()
            if it >= a.warmup:
                ms[arm].append(e0.elapsed_time(e1))
    name, power = card()
    peak = bench.HBM_PEAK_GBS
    for arm in arms:
        t = float(np.median(ms[arm]))
        alg = in_bytes + img_bytes[arm]
        kind, mode = arm
        print(json.dumps({"workload": "device encoder, cfg5 columns", "encoding": kind, "stream_mode": mode, "rows": n, "rows_per_block": a.rows_per_block,
                          "n_blocks": nb[arm], "ms": round(t, 3), "ms_min": round(min(ms[arm]), 3), "ms_max": round(max(ms[arm]), 3),
                          "rows_per_s": n / t * 1e3, "in_bytes": in_bytes, "image_bytes": img_bytes[arm],
                          "alg_gbps": round(alg / t / 1e6, 1), "peak_gbps": peak, "frac": round(alg / t / 1e6 / peak, 3),
                          "gpu": name, "power_limit": power, "writer_verified": a.verify,
                          "note": "event-timed around obgpu_encode_columns_%s (includes its allocation + the 64 KB table upload)"
                                  % ("cs_ex" if kind.startswith("cs") else "ex")}))


if __name__ == "__main__":
    main()
