"""The device CS encoder with integer stream codecs (obgpu_encode_columns_cs_ex / obgpu_merge_result_encode_cs_ex): under every
stream mode the blocks equal, byte for byte, what obgpu_writer_encode_table writes for the same rows and per-column encodings
after obgpu_writer_set_cs_stream_encoding(mode): image, offsets, sizes, header and payload checksums."""
import numpy as np
import pytest

import oracle_binding as ora
from test_gpu_device_encoder_cs import INT, DICT, AUTO, TYPES, I64_MIN, I64_MAX, _col, _type_range, assert_same_image

pytestmark = pytest.mark.gpu

MODES = (0, 1, 2, 3, 4, 5, 6, 8)


@pytest.fixture(autouse=True)
def writer_mode():
    """The writer's CS stream mode is process-wide: each case sets it through writer_table, and mode 1 is restored afterwards."""
    from oceanbase_b200 import capi
    yield
    capi.lib.obgpu_writer_set_cs_stream_encoding(1)


def _ctx():
    import oceanbase_b200 as ob
    return ob.ScanContext(0)


def writer_table(cols, encs, rpb, rk, mode, align=128):
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, encode_table
    assert capi.lib.obgpu_writer_set_cs_stream_encoding(mode) == 0
    return encode_table([Column(t, e, v, nulls=nl) for (t, v, nl), e in zip(cols, encs)], rpb, rowkey_cnt=rk, align=align)


def device_encode(ctx, cols, encs, rpb, rk, mode, align=128):
    import torch
    from oceanbase_b200 import compaction
    keep, dcols = [], []
    for (t, v, nl) in cols:
        dv = torch.from_numpy(np.ascontiguousarray(v)).cuda()
        dn = torch.from_numpy(np.ascontiguousarray(nl)).cuda() if nl is not None else None
        keep += [dv, dn]
        dcols.append((dv.data_ptr(), dn.data_ptr() if dn is not None else None, t, False))
    return compaction.encode_columns(ctx, dcols, len(cols[0][1]), rpb, rowkey_cnt=rk, align=align, keep=keep, encodings=encs, cs=True,
                                     stream_mode=mode)


def check(ctx, cols, encs, rpb, mode, rk=0, align=128):
    table = writer_table(cols, encs, rpb, rk, mode, align)
    enc = device_encode(ctx, cols, encs, rpb, rk, mode, align)
    assert_same_image(enc, table)
    return table, enc


def _walk(rng, n, steps, t):
    lo, hi = _type_range(t)
    v = np.cumsum(rng.choice(np.asarray(steps, dtype=np.int64), n)).astype(np.int64)
    if t == 5:
        return v
    if t in (6, 7, 9, 10):
        return (v.astype(np.uint64) % np.uint64(hi)).astype(np.uint64)
    return (v - lo) % (hi - lo) + lo


def shaped_columns(n, seed):
    """Columns whose streams cover the codecs' edges: widths 1 / 2 / 4 / 8 with a base and with a NULL replacement, monotonic
    and decreasing streams, RLE runs around 18 and 273 zero deltas, deltas at each tier edge and above 45 bits, trailing zero
    runs, constant blocks (candidates tie), and full-width random data (every codec falls back to RAW)."""
    rng = np.random.default_rng(seed)
    runs = np.concatenate([np.full(r, k, dtype=np.int64) for k, r in enumerate([18, 19, 20, 273, 274, 275, 1, 2] * (n // 900 + 1))])[:n]
    edges = [0, 0, 1, -1, 2, -2, 3, -3, 4, 15, 16, -16, -17, 31, 32, 255, 256, 511, 512, 1023, 1024, 2047, 2048, 65535, 65536,
             (1 << 18) - 1, 1 << 18, 1 << 19, 1 << 30, 1 << 44, 1 << 45, 1 << 46, -(1 << 47), 1 << 52]
    cols = [
        _col(5, np.arange(n) * 3 + 11),                                      # monotonic, no base: XOR skipped
        _col(5, np.arange(n)[::-1] - 40, rng.random(n) < 0.02),              # decreasing, base, NULL replacement
        _col(1, rng.integers(-128, 127, n), rng.random(n) < 0.05),           # width 1 with base
        _col(6, rng.integers(0, 255, n)),                                    # width 1
        _col(2, _walk(rng, n, [0, 1, -1, 15, 16, -17, 300], 2)),             # width 2 walk
        _col(7, np.sort(rng.integers(0, 1 << 16, n)).astype(np.uint64)),     # width 2 monotonic
        _col(4, _walk(rng, n, [0, 0, 0, 31, 32, -511, 512, 65536, -70000], 4), rng.random(n) < 0.01),   # width 4 tiers
        _col(9, rng.integers(0, 1 << 32, n).astype(np.uint64)),              # width 4 random
        _col(5, _walk(rng, n, edges, 5)),                                    # width 8: every tier edge, wide deltas
        _col(5, rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)),          # full width random: RAW everywhere
        _col(10, rng.integers(0, 1 << 62, n).astype(np.uint64) | np.uint64(1 << 63)),   # width 8 unsigned, high bit set
        _col(5, runs),                                                       # RLE runs 18 / 19 / 273 / 274
        _col(5, runs * 3 + np.arange(n)),                                    # DD runs: a constant stride
        _col(5, np.full(n, 5)),                                              # constant: a run over the whole block, ties
        _col(5, np.r_[rng.integers(0, 100, n // 2), np.full(n - n // 2, 7)]),   # trailing zero run
        _col(3, np.zeros(n), np.tile([0, 0, 1], n // 3 + 1)[:n]),            # NULL replaced, all-zero stream otherwise
    ]
    return cols


@pytest.mark.parametrize("enc", [INT, DICT, AUTO])
@pytest.mark.parametrize("mode", MODES)
def test_every_mode_every_type(mode, enc):
    """Every stream mode x every integer obj type x CS_INTEGER / CS_INT_DICT / CS_AUTO, against the host writer at that mode."""
    ctx = _ctx()
    rng = np.random.default_rng(100 + mode)
    n = 3_000
    cols = []
    for t in TYPES:
        lo, hi = _type_range(t)
        cols.append(_col(t, rng.integers(lo, hi, n), rng.random(n) < 0.03))
        cols.append(_col(t, rng.integers(lo, lo + 9, n)))
        cols.append(_col(t, np.sort(rng.integers(lo, hi, n))))
    check(ctx, cols, [enc] * len(cols), 500, mode)[1].free()


@pytest.mark.parametrize("mode", MODES)
def test_stream_shapes(mode):
    ctx = _ctx()
    cols = shaped_columns(6_000, 7)
    for enc, rpb, nc in ((INT, 1_025, 16), (INT, 700, 16), (DICT, 700, 16), (DICT, 1_025, 8)):   # blocks that fit one CTA
        check(ctx, cols[:nc], [enc] * nc, rpb, mode)[1].free()


@pytest.mark.parametrize("rpb", [1, 2, 3, 4, 127, 128, 129, 256, 257, 1_023, 1_024, 1_025, 2_600, 4_500])
def test_stream_lengths(rpb):
    """Stream lengths around the chunk (128) and sample (1 024, 4 values) boundaries, in every mode; a ragged last block."""
    ctx = _ctx()
    cols = shaped_columns(2 * rpb + (rpb + 1) // 2, 11)
    n_int, n_dict = (9, 4) if rpb <= 1_025 else (3, 1 if rpb <= 2_600 else 0)   # blocks that fit one CTA
    for mode in MODES:
        check(ctx, cols[:n_int], [INT] * n_int, rpb, mode)[1].free()
        if n_dict:
            check(ctx, cols[8:8 + n_dict], [DICT] * n_dict, rpb, mode)[1].free()


@pytest.mark.parametrize("mode", MODES)
def test_const_form_ref_streams(mode):
    """Dictionary ref streams in the const form (0, 1, 64 exceptions: 2, 4 and 130 values, forced codecs encode them too) and
    plain."""
    ctx = _ctx()
    n, rpb = 3_000, 1_000
    rng = np.random.default_rng(5)
    cols = []
    for exc in (0, 1, 64, 99, 300):
        v = np.full(n, -42, dtype=np.int64)
        for b in range(n // rpb):
            rows = rng.choice(rpb, exc, replace=False) + b * rpb
            v[rows] = rng.integers(0, 1 << 20, exc)
        cols.append(_col(5, v))
    nl = np.zeros(n, dtype=np.uint8)
    nl[::50] = 1
    cols.append(_col(5, np.full(n, 3), nl))   # the NULL ref as exception
    check(ctx, cols, [DICT] * len(cols), rpb, mode)[1].free()


def test_codecs_are_written():
    """Detection does pick codecs on shaped data (the images are not all RAW), and each forced mode writes its own type."""
    ctx = _ctx()
    cols = shaped_columns(4_000, 3)
    for mode in MODES:
        _, enc = check(ctx, cols, [INT] * len(cols), 1_000, mode)
        img, off, sz = enc.fetch()
        b = np.asarray(img[off[0]:off[0] + sz[0]])
        # the first column's stream meta (monotonic, no NULL): right behind the column headers
        meta = 64 + 12 + 4 * len(cols)
        got = int(b[meta + 2])
        if mode == 1:
            assert got == 1
        elif mode != 0:
            assert got in (mode, 1)
        else:
            assert got != 1
        enc.free()


def test_closed_loop_scan_and_compress():
    """Mode-0 blocks re-open from the device image and scan to the input columns; compressed with LZ4 and zstd_1.3.8 on the
    device they equal the writer's compressed table and scan the same; column checksums equal mode 1's."""
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import TableImage, compress_table
    ctx = _ctx()
    rng = np.random.default_rng(12)
    n = 20_000
    cols = [_col(5, np.arange(n) * 2 + 5), _col(5, rng.integers(0, 40, n), rng.random(n) < 0.07),
            _col(5, np.repeat(rng.integers(-(1 << 40), 1 << 40, n // 30 + 1), 30)[:n]), _col(4, np.full(n, 11)),
            _col(5, np.cumsum(rng.integers(-3, 4, n)))]
    encs = [INT, AUTO, DICT, AUTO, INT]
    table, enc = check(ctx, cols, encs, 700, 0, rk=1)
    raw = device_encode(ctx, cols, encs, 700, 1, 1)
    assert np.array_equal(enc.column_checksums(), raw.column_checksums())
    assert enc.info().image_size < raw.info().image_size
    raw.free()
    img, off, sz = enc.fetch()
    d_img, _, _ = enc.device_image()
    flt = ob.White(0, ob.WHITE_OP_GE, [0])
    proj = list(range(len(cols)))

    def scan(b):
        r = b.scan(flt, proj)
        assert r.selected_rows == n
        for i, (t, v, nl) in enumerate(cols):
            d, _, _ = r.fetch_col(i)
            d = d[:n]
            keep = np.ones(n, bool) if nl is None else ~nl.astype(bool)
            exp = v[keep]
            got = d.view(np.int64)[keep] if d.dtype.itemsize == 8 else d[keep].astype(np.int64)
            assert np.array_equal(got, exp.astype(np.int64)), i
    dev = ob.PageBatch(ctx, TableImage(img, off, sz, n, len(cols)), device_image_ptr=d_img, image_size=img.size)
    scan(dev)
    dev.close()
    for comp in (2, 6):
        c = enc.compress(comp)
        g_img, g_off, g_sz = c.fetch()
        st = compress_table(table, comp, align=128)
        assert np.array_equal(g_img, np.asarray(st.image)), comp
        cb = ob.PageBatch(ctx, TableImage(g_img, g_off, g_sz, n, len(cols)), device_image_ptr=c.image.data_ptr(),
                          image_size=c.image_size, compressor=comp)
        scan(cb)
        cb.close()
    for b in (0, len(off) - 1):
        assert ora.Block(img[off[b]:off[b] + sz[b]].copy()).verify_checksums() == 0, b
    enc.free()


def test_merge_result_mode0():
    """merge -> encode_merge_result(cs=True, stream_mode=0) and co_merge_write: equal to the host writer at mode 0."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction
    from oceanbase_b200.sstable import Column, encode_table
    ctx = _ctx()
    rng = np.random.default_rng(9)
    runs = []
    for r in range(3):
        n = 6_000
        key = np.sort(rng.choice(40_000, size=n, replace=False)).astype(np.int64)
        cols = [Column(capi.OBJ_INT, INT, key), Column(capi.OBJ_INT, DICT, rng.integers(-5, 5, size=n, dtype=np.int64)),
                Column(capi.OBJ_INT, INT, rng.integers(0, 1 << 40, size=n, dtype=np.int64), nulls=(rng.random(n) < 0.1).astype(np.uint8))]
        runs.append(encode_table(cols, 700, rowkey_cnt=1))
    batches = [ob.PageBatch(ctx, t) for t in runs]
    res = compaction.merge_batches(ctx, batches, 0, None, [1, 2])
    key, _ = res.fetch(-1)
    payload = [res.fetch(c) for c in range(2)]
    assert capi.lib.obgpu_writer_set_cs_stream_encoding(0) == 0

    def host(cg, encodings, rpb):
        hc = []
        for c in cg:
            v, nl = (key, None) if c == -1 else payload[c]
            hc.append(Column(capi.OBJ_INT, encodings[c], v, nulls=nl if nl is not None and nl.any() else None))
        return encode_table(hc, rpb, rowkey_cnt=1 if cg[0] == -1 else 0)
    one = compaction.encode_merge_result(res, [-1, 0, 1], [capi.OBJ_INT] * 3, 512, encodings=[INT, DICT, AUTO], cs=True, stream_mode=0)
    assert_same_image(one, host([-1, 0, 1], {-1: INT, 0: DICT, 1: AUTO}, 512))
    one.free()
    groups = [[-1, 0], [1]]
    encodings = {-1: INT, 0: AUTO, 1: INT}
    for cg, enc in zip(groups, compaction.co_merge_write(res, groups, {c: capi.OBJ_INT for c in (-1, 0, 1)}, 900, encodings=encodings,
                                                         cs=True, stream_mode=0)):
        assert_same_image(enc, host(cg, encodings, 900))
        enc.free()
    for b in batches:
        b.close()


def test_mode1_ex_equals_the_old_entry_point():
    import ctypes as C
    import torch
    from oceanbase_b200 import capi, compaction
    ctx = _ctx()
    rng = np.random.default_rng(4)
    n = 5_000
    cols = shaped_columns(n, 2)
    dv = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for _, v, _ in cols]
    dn = [torch.from_numpy(np.ascontiguousarray(nl)).cuda() if nl is not None else None for _, _, nl in cols]
    arr = compaction._encode_cols([(v.data_ptr(), None if m is None else m.data_ptr(), t, False) for v, m, (t, _, _) in zip(dv, dn, cols)])
    encs = np.asarray(rng.choice([INT, DICT, AUTO], len(cols)), dtype=np.int32)
    h_old, h_new = C.c_void_p(), C.c_void_p()
    assert capi.lib.obgpu_encode_columns_cs(ctx._h, arr, encs.ctypes.data, len(cols), 0, n, 777, 256, C.byref(h_old)) == 0
    assert capi.lib.obgpu_encode_columns_cs_ex(ctx._h, arr, encs.ctypes.data, len(cols), 0, n, 777, 256, 1, C.byref(h_new)) == 0
    a, b = compaction.Encoded(ctx, h_old, len(cols)), compaction.Encoded(ctx, h_new, len(cols))
    for x, y in zip(a.fetch(), b.fetch()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.column_checksums(), b.column_checksums())
    a.free()
    b.free()


def test_refusals_and_ctx_reuse():
    from oceanbase_b200 import capi, compaction
    ctx = _ctx()
    cols = [_col(5, np.arange(100))]
    before = ctx.launch_count
    for mode in (7, 9, -1, 100):
        with pytest.raises(capi.ObGpuError) as ei:
            device_encode(ctx, cols, [INT], 10, 0, mode)
        assert ei.value.code == capi.OB_INVALID_ARGUMENT
    assert ctx.launch_count == before
    with pytest.raises(ValueError):
        compaction.encode_columns(ctx, [(0, None, 5, False)], 100, 10, stream_mode=0)
    check(ctx, cols, [INT], 10, 0)[1].free()


def _largest_rpb(ctx, cols, encs, mode):
    from oceanbase_b200 import capi

    def fits(r):
        try:
            device_encode(ctx, cols, encs, r, 1, mode).free()
            return True
        except capi.ObGpuError as e:
            assert e.code == capi.OB_NOT_SUPPORTED
            return False
    lo, hi = 1, 1 << 16
    assert fits(lo) and not fits(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    return lo


def test_shared_memory_limit():
    """The largest rows_per_block of the cfg5 shape with stream codecs (the CsCodec records, chunk histograms, const-form refs
    and chunk sizes): encoded right there in mode 0, one row more refused before any launch with the ctx still usable."""
    ctx = _ctx()
    rng = np.random.default_rng(3)
    n = 70_000
    cols = [_col(5, np.arange(n) * 3 + 7), _col(5, rng.integers(0, 1 << 33, n)), _col(5, rng.integers(-(1 << 62), 1 << 62, n)),
            _col(5, rng.integers(0, 1 << 13, n), rng.random(n) < 0.05)]
    got = {}
    for name, encs in (("int", [INT] * 4), ("auto", [AUTO] * 4)):
        lo = _largest_rpb(ctx, cols, encs, 0)
        print(f"largest CS rows_per_block with stream codecs, cfg5 shape, {name}:", lo)
        check(ctx, cols, encs, lo, 0, rk=1)[1].free()
        got[name] = lo
    assert got == {"int": 6_660, "auto": 2_898}, got


def test_launch_count_does_not_depend_on_blocks():
    ctx = _ctx()
    counts = []
    for blocks in (10, 20_000):
        cols = [_col(5, np.arange(blocks * 7)), _col(4, np.arange(blocks * 7) % 5)]
        before = ctx.launch_count
        enc = device_encode(ctx, cols, [INT, AUTO], 7, 1, 0)
        enc.info()
        counts.append(ctx.launch_count - before)
        enc.free()
    assert counts[0] == counts[1] == 1, counts


def test_seeded_random_differential():
    ctx = _ctx()
    rng = np.random.default_rng(2024)
    for case in range(24):
        mode = MODES[case % len(MODES)]
        n = int(rng.integers(1, 5_000))
        rpb = min(int(rng.choice([1, 5, 64, 128, 300, 1_000, 1_500, n])), 1_500)
        cols, encs = [], []
        for _ in range(int(rng.integers(1, 7))):
            t = int(rng.choice(TYPES))
            lo, hi = _type_range(t)
            shape = int(rng.integers(0, 4))
            if shape == 0:
                v = rng.integers(lo, hi, n)
            elif shape == 1:
                v = np.sort(rng.integers(lo, hi, n))
            elif shape == 2:
                v = np.repeat(rng.integers(lo, hi, n // 20 + 1), 20)[:n]
            else:
                v = rng.integers(lo, min(hi, lo + int(rng.integers(1, 40))), n)
            nf = float(rng.choice([0.0, 0.0, 0.01, 0.2, 1.0]))
            cols.append(_col(t, v, (rng.random(n) < nf) if nf > 0 else None))
            encs.append(int(rng.choice([INT, DICT, AUTO])))
        check(ctx, cols, encs, rpb, mode)[1].free()
