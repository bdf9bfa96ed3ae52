"""The device encoder for CS_ENCODING_ROW_STORE tables (obgpu_encode_columns_cs / obgpu_merge_result_encode_cs): per block and
per column CS_INTEGER or CS_INT_DICT (CS_AUTO: the writer's choose_cs_auto_encoding), byte for byte the blocks
obgpu_writer_encode_table writes with the same per-column encodings and RAW integer streams: image, offsets, sizes, column
checksums."""
import numpy as np
import pytest

import oracle_binding as ora

pytestmark = pytest.mark.gpu

INT, DICT, AUTO = 16, 17, 33
TYPES = (1, 2, 3, 4, 5, 6, 7, 9, 10, 17, 19, 21)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(autouse=True)
def raw_streams():
    """The writer's CS stream mode is process-wide: RAW streams (mode 1) for the comparison, and mode 1 again afterwards."""
    from oceanbase_b200 import capi
    assert capi.lib.obgpu_writer_set_cs_stream_encoding(1) == 0
    yield
    capi.lib.obgpu_writer_set_cs_stream_encoding(1)


def _ctx():
    import oceanbase_b200 as ob
    return ob.ScanContext(0)


def _col(t, v, nl=None):
    return (t, np.asarray(v, dtype=np.uint64 if np.asarray(v).dtype == np.uint64 else np.int64).view(np.int64),
            None if nl is None else np.asarray(nl, dtype=np.uint8))


def writer_table(cols, encs, rpb, rk, align=128):
    from oceanbase_b200.sstable import Column, encode_table
    return encode_table([Column(t, e, v, nulls=nl) for (t, v, nl), e in zip(cols, encs)], rpb, rowkey_cnt=rk, align=align)


def device_encode(ctx, cols, encs, rpb, rk, align=128):
    import torch
    from oceanbase_b200 import compaction
    keep, dcols = [], []
    for (t, v, nl) in cols:
        dv = torch.from_numpy(np.ascontiguousarray(v)).cuda()
        dn = torch.from_numpy(np.ascontiguousarray(nl)).cuda() if nl is not None else None
        keep += [dv, dn]
        dcols.append((dv.data_ptr(), dn.data_ptr() if dn is not None else None, t, False))
    return compaction.encode_columns(ctx, dcols, len(cols[0][1]), rpb, rowkey_cnt=rk, align=align, keep=keep, encodings=encs, cs=True)


def assert_same_image(enc, table):
    img, off, sz = enc.fetch()
    info = enc.info()
    assert info.n_blocks == table.n_blocks
    assert info.n_host_blocks == 0
    assert np.array_equal(off, np.asarray(table.offsets)), "block offsets differ"
    assert np.array_equal(sz, np.asarray(table.sizes)), "block sizes differ"
    want = np.asarray(table.image)
    assert img.size == want.size, (img.size, want.size)
    if not np.array_equal(img, want):
        bad = int(np.nonzero(img != want)[0][0])
        blk = int(np.searchsorted(off, bad, side="right") - 1)
        raise AssertionError(f"first differing byte {bad} (block {blk}, byte {bad - off[blk]} of {sz[blk]})")


def check(ctx, cols, encs, rpb, rk=0, align=128):
    table = writer_table(cols, encs, rpb, rk, align)
    enc = device_encode(ctx, cols, encs, rpb, rk, align)
    assert_same_image(enc, table)
    img, off, sz = enc.fetch()
    for b in sorted({0, len(off) // 2, len(off) - 1}):
        assert ora.Block(img[off[b]:off[b] + sz[b]].copy()).verify_checksums() == 0, b
    o = ora.oracle()
    got = enc.column_checksums()
    for c, (t, v, nl) in enumerate(cols):
        dl = 1 if t == 21 else (4 if t == 19 else 8)
        v = np.ascontiguousarray(v)
        assert int(got[c]) == o.ora_column_checksum(v.ctypes.data, nl.ctypes.data if nl is not None else None, len(v), dl), c
    return table, enc


def cs_layout(block, n_cols):
    """(column types, column attrs, stream-offsets width) of one CS block."""
    b = np.asarray(block)
    types = [int(b[64 + 12 + 4 * c + 1]) for c in range(n_cols)]
    attrs = [int(b[64 + 12 + 4 * c + 2]) for c in range(n_cols)]
    so_len = int(b[70:74].view(np.uint32)[0])
    cnt = int(b[74:76].view(np.uint16)[0])
    return types, attrs, ((so_len - 5) // cnt if cnt else 0)


def _type_range(t):
    return {1: (-128, 128), 2: (-(1 << 15), 1 << 15), 3: (-(1 << 23), 1 << 23), 4: (-(1 << 31), 1 << 31), 5: (-(1 << 62), 1 << 62),
            6: (0, 256), 7: (0, 1 << 16), 9: (0, 1 << 32), 10: (0, 1 << 62), 17: (-(1 << 40), 1 << 40), 19: (-50_000, 50_000),
            21: (0, 120)}[t]


def shapes():
    """name -> (cols, rows_per_block, rowkey_cnt)"""
    rng = np.random.default_rng(31)
    n = 3_000
    S = {}
    cols = []
    for t in TYPES:
        lo, hi = _type_range(t)
        cols.append(_col(t, rng.integers(lo, hi, n), rng.random(n) < 0.03))
        cols.append(_col(t, rng.integers(lo, lo + 9, n)))
    S["types"] = (cols, 500, 0)
    # CS_INTEGER NULL replacement: every branch in every block of 100 rows (the extremes and a NULL in each block)
    m = 100

    def tiled(extremes, fill, t=5):
        v = np.tile(np.array(list(extremes) + [fill] * (m - len(extremes)), dtype=np.uint64 if t in (6, 7, 9, 10) else np.int64), n // m)
        nl = np.tile(np.concatenate([np.zeros(len(extremes)), [1], np.zeros(m - len(extremes) - 1)]), n // m)
        return _col(t, v, nl)
    S["null_branches"] = ([tiled([0, 77], 5), tiled([0, I64_MAX], 5), tiled([I64_MIN, 9], 5), tiled([I64_MIN, I64_MAX], 5),
                           tiled([-50, 50], 3), tiled([-128, 127], 1, 1), tiled([0, 127], 1, 1), tiled([-128, 3], 1, 1),
                           tiled([0, 255], 7, 6), tiled([0, 10], 7, 6), tiled([5, 10], 7, 6), tiled([0, (1 << 64) - 1], 3, 10),
                           tiled([3, 1 << 40], 9, 10), _col(5, np.zeros(n), np.ones(n)), _col(6, np.zeros(n), np.ones(n)),
                           _col(1, np.full(n, -5)), _col(5, np.full(n, 9), np.tile([0, 1, 0], n // 3))], m, 0)
    S["negative_dict"] = ([_col(5, rng.integers(-20, 5, n)), _col(1, rng.integers(-128, -100, n), rng.random(n) < 0.1),
                           _col(2, rng.choice([-30_000, -1, 0, 30_000], n)), _col(4, rng.integers(-(1 << 31), -(1 << 31) + 40, n)),
                           _col(5, rng.choice([I64_MIN, -7, I64_MAX], n)), _col(3, rng.integers(-9, 9, n), rng.random(n) < 0.4)], 500, 1)
    # datums that are not sign-extended: the writer keys a signed column on the full datum, its AUTO estimate on the store image
    S["not_sign_extended"] = ([_col(1, rng.choice([200, -56, 3, -3], n)), _col(2, rng.choice([40_000, -25_536, 7], n), rng.random(n) < 0.1),
                               _col(4, rng.choice([(1 << 32) - 1, -1, 1 << 31], n))], 300, 0)
    S["ragged"] = ([_col(5, np.arange(2_001) * 2), _col(5, rng.integers(0, 3, 2_001), rng.random(2_001) < 0.1),
                    _col(10, rng.integers(0, 1 << 62, 2_001).astype(np.uint64))], 133, 1)
    return S


SHAPES = shapes()


@pytest.mark.parametrize("enc", [INT, DICT, AUTO])
@pytest.mark.parametrize("name", list(SHAPES))
def test_cs_blocks_equal_the_host_writer(name, enc):
    ctx = _ctx()
    cols, rpb, rk = SHAPES[name]
    check(ctx, cols, [enc] * len(cols), rpb, rk)[1].free()


def test_integer_null_branches_are_covered():
    """The null_branches shape takes the NULL bitmap (signed and unsigned, both ends of the type range used) and replaces NULL
    in the other columns."""
    cols, rpb, rk = SHAPES["null_branches"]
    t = writer_table(cols, [INT] * len(cols), rpb, rk)
    _, attrs, _ = cs_layout(t.block(0), len(cols))
    assert [i for i, a in enumerate(attrs) if a & 0x2] == [3, 5, 8, 11], attrs


def _const_block(rng, n, exc, ref_null=False):
    v = np.full(n, 1000, dtype=np.int64)
    nl = np.zeros(n, np.uint8)
    pos = rng.choice(n, exc, replace=False)
    v[pos] = rng.integers(-5, 5, exc) * 7
    if ref_null:
        nl[:] = 1
        nl[pos] = 0
    return v, nl


@pytest.mark.parametrize("enc", [DICT, AUTO])
def test_const_ref_boundaries(enc):
    """put_dict_ref_stream's const form at exc 0, 64 at n = 650 (the smallest n where 64 < n * 10 / 100), 65, and exactly 10 %,
    and with NULL as the constant."""
    ctx = _ctx()
    rng = np.random.default_rng(5)
    for n, exc, ref_null in ((650, 0, False), (650, 64, False), (650, 65, False), (640, 64, False), (650, 64, True), (650, 0, True),
                             (300, 29, False)):
        v, nl = _const_block(rng, n, exc, ref_null)
        cols = [_col(5, np.tile(v, 3), np.tile(nl, 3)), _col(5, np.tile(v, 3))]
        check(ctx, cols, [enc, enc], n, 0)[1].free()


def test_auto_picks_both_sides():
    """CS_AUTO over a sweep of distinct counts and value ranges: the writer picks INTEGER and INT_DICT, the device the same."""
    ctx = _ctx()
    rng = np.random.default_rng(8)
    n, rpb = 4_000, 400
    cols = []
    for d in (2, 20, 120, 199, 200, 201, 260, 399):
        for bits in (6, 9, 40):
            vals = rng.choice(rng.integers(0, 1 << bits, 4 * d), d, replace=True)
            cols.append(_col(5, vals[rng.integers(0, d, n)], rng.random(n) < 0.02 if bits == 9 else None))
    table, enc = check(ctx, cols, [AUTO] * len(cols), rpb, 0)
    seen = set()
    for b in range(table.n_blocks):
        seen |= set(cs_layout(table.block(b), len(cols))[0])
    assert seen == {0, 2}, seen
    enc.free()


@pytest.mark.parametrize("rpb", [1, 2, 7, 133, 500])
def test_rows_per_block_and_short_last_block(rpb):
    ctx = _ctx()
    rng = np.random.default_rng(rpb)
    n = 1_003 if rpb > 2 else 41
    cols = [_col(5, np.arange(n) * 5), _col(4, rng.integers(-9, 9, n), rng.random(n) < 0.2), _col(6, rng.integers(0, 256, n))]
    for e in ([INT] * 3, [DICT] * 3, [AUTO] * 3, [INT, DICT, AUTO]):
        check(ctx, cols, e, rpb, 1)[1].free()


def test_stream_offset_widths():
    ctx = _ctx()
    rng = np.random.default_rng(4)
    for rpb, cols_n, want in ((7, 1, 1), (500, 1, 2), (9_000, 1, 4)):
        n = rpb * 2 + 3
        cols = [_col(5, rng.integers(-(1 << 62), 1 << 62, n)) for _ in range(cols_n)]
        table, enc = check(ctx, cols, [INT] * cols_n, rpb, 0)
        assert cs_layout(table.block(0), cols_n)[2] == want
        enc.free()


@pytest.mark.parametrize("align", [16, 32, 128, 512, 4096])
def test_alignments(align):
    ctx = _ctx()
    cols, rpb, rk = SHAPES["negative_dict"]
    check(ctx, cols, [INT, DICT, AUTO, INT, AUTO, DICT], rpb, rk, align=align)[1].free()


@pytest.mark.parametrize("n_cols,rk", [(1, 0), (1, 1), (2, 2), (33, 1), (64, 0), (64, 2)])
def test_column_counts(n_cols, rk):
    ctx = _ctx()
    rng = np.random.default_rng(n_cols)
    n = 1_500
    cols = [_col(int(rng.choice(TYPES)), rng.integers(0, 1 << int(rng.integers(1, 7)), n), rng.random(n) < 0.05 if c % 3 == 1 else None)
            for c in range(n_cols)]
    check(ctx, cols, [(INT, DICT, AUTO)[c % 3] for c in range(n_cols)], 250, rk)[1].free()


def test_seeded_random_differential():
    ctx = _ctx()
    rng = np.random.default_rng(2025)
    for it in range(12):
        n = int(rng.integers(1, 5_000))
        rpb = int(rng.choice([1, 2, 7, 64, 133, 500, 1_000]))
        cols, encs = [], []
        for c in range(int(rng.integers(1, 12))):
            t = int(rng.choice(TYPES))
            lo, hi = _type_range(t)
            kind = int(rng.integers(0, 5))
            if kind == 0:
                v = rng.integers(lo, hi, n)
            elif kind == 1:
                v = rng.integers(-3, 4, n) * int(rng.integers(1, 1 << 20))
            elif kind == 2:
                run = int(rng.integers(1, 40))
                v = np.repeat(rng.integers(-1000, 1000, n // run + 1), run)[:n]
            elif kind == 3:
                v = np.full(n, int(rng.integers(-100, 100)))
                k = int(rng.integers(0, 70))
                v[rng.integers(0, n, k)] = rng.integers(-100, 100, k)
            else:
                v = np.cumsum(rng.integers(0, 1000, n)) - int(rng.integers(0, 1 << 30))
            if t not in (1, 2, 3, 4, 5, 17, 19):   # unsigned: non-negative values
                v = np.abs(v)
            nf = float(rng.choice([0.0, 0.0, 0.01, 0.2, 0.6, 1.0]))
            nl = (rng.random(n) < nf) if nf > 0 else None
            cols.append(_col(t, v, nl))
            encs.append(int(rng.choice([INT, DICT, AUTO, AUTO])))
        check(ctx, cols, encs, rpb, 0)[1].free()


def test_reopen_scan_and_compress():
    """CS blocks re-open from the device image as a page batch that scans like the writer's table; compressed on the device with
    LZ4 and zstd_1.3.8 they open through obgpu_batch_open_compressed and scan the same."""
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import TableImage, compress_table
    ctx = _ctx()
    rng = np.random.default_rng(12)
    n = 20_000
    cols = [_col(5, np.arange(n) * 2 + 5), _col(5, rng.integers(0, 40, n), rng.random(n) < 0.07),
            _col(5, np.repeat(rng.integers(-(1 << 40), 1 << 40, n // 30 + 1), 30)[:n]), _col(4, np.full(n, 11))]
    table, enc = check(ctx, cols, [INT, AUTO, DICT, AUTO], 700, 1)
    img, off, sz = enc.fetch()
    d_img, _, _ = enc.device_image()
    flt = ob.And([ob.White(1, ob.WHITE_OP_LT, [30]), ob.White(0, ob.WHITE_OP_GE, [1000])])
    want = (~cols[1][2].astype(bool)) & (cols[1][1] < 30) & (cols[0][1] >= 1000)

    def scan(b):
        r = b.scan(flt, [0, 2, 3])
        assert r.selected_rows == int(want.sum())
        out = []
        for i, c in enumerate((0, 2, 3)):
            d, _, _ = r.fetch_col(i)
            d = d[:r.selected_rows]
            exp = cols[c][1][want]
            assert np.array_equal(d.view(np.int64), exp) if d.dtype.itemsize == 8 else np.array_equal(d, exp.astype(d.dtype)), c
            out.append(d.copy())
        return out
    dev = ob.PageBatch(ctx, TableImage(img, off, sz, n, 4), device_image_ptr=d_img, image_size=img.size)
    ref = ob.PageBatch(ctx, table)
    got, exp = scan(dev), scan(ref)
    assert all(np.array_equal(a, b) for a, b in zip(got, exp))
    dev.close()
    ref.close()
    for comp in (2, 6):
        c = enc.compress(comp)
        g_img, g_off, g_sz = c.fetch()
        st = compress_table(table, comp, align=128)
        assert np.array_equal(g_off, np.asarray(st.offsets)) and np.array_equal(g_sz, np.asarray(st.sizes)), comp
        assert np.array_equal(g_img, np.asarray(st.image)), comp
        cb = ob.PageBatch(ctx, TableImage(g_img, g_off, g_sz, n, 4), device_image_ptr=c.image.data_ptr(), image_size=c.image_size,
                          compressor=comp)
        assert all(np.array_equal(a, b) for a, b in zip(scan(cb), exp))
        cb.close()
    enc.free()


def test_merge_result_column_groups():
    """merge -> co_merge_write(cs=True): every group equals the host writer in CS mode over the merged rows fetched back."""
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
                Column(capi.OBJ_INT, INT, rng.integers(0, 1 << 40, size=n, dtype=np.int64), nulls=(rng.random(n) < 0.1).astype(np.uint8)),
                Column(capi.OBJ_INT, AUTO, np.full(n, 77, dtype=np.int64))]
        runs.append(encode_table(cols, 700, rowkey_cnt=1))
    batches = [ob.PageBatch(ctx, t) for t in runs]
    res = compaction.merge_batches(ctx, batches, 0, None, [1, 2, 3])
    key, _ = res.fetch(-1)
    payload = [res.fetch(c) for c in range(3)]
    groups = [[-1, 0, 1, 2], [0], [1], [2, 0]]
    types = {c: capi.OBJ_INT for c in (-1, 0, 1, 2)}
    encodings = {-1: INT, 0: DICT, 1: AUTO, 2: AUTO}
    encs = compaction.co_merge_write(res, groups, types, rows_per_block=900, encodings=encodings, cs=True)
    for cg, enc in zip(groups, encs):
        host_cols = []
        for c in cg:
            v, nl = (key, None) if c == -1 else payload[c]
            host_cols.append(Column(capi.OBJ_INT, encodings[c], v, nulls=nl if nl is not None and nl.any() else None))
        table = encode_table(host_cols, 900, rowkey_cnt=1 if cg[0] == -1 else 0)
        assert_same_image(enc, table)
        enc.free()
    one = compaction.encode_merge_result(res, [-1, 1], [capi.OBJ_INT] * 2, 512, cs=True)
    table = encode_table([Column(capi.OBJ_INT, INT, key), Column(capi.OBJ_INT, INT, payload[1][0],
                                                                  nulls=payload[1][1] if payload[1][1].any() else None)], 512, rowkey_cnt=1)
    assert_same_image(one, table)
    one.free()


def test_refusals_and_ctx_reuse():
    import torch
    from oceanbase_b200 import capi, compaction
    ctx = _ctx()
    cols = [_col(5, np.arange(100))]

    def refused(code, encs=None, **kw):
        with pytest.raises(capi.ObGpuError) as ei:
            args = dict(cols=cols, encs=encs, rpb=10, rk=0)
            args.update(kw)
            device_encode(ctx, args["cols"], args["encs"], args["rpb"], args["rk"], args.get("align", 128))
        assert ei.value.code == code
    for e in (capi.ENC_RAW, capi.ENC_AUTO, capi.ENC_DICT, capi.ENC_CONST, capi.ENC_CS_STRING, capi.ENC_CS_STR_DICT):
        refused(capi.OB_NOT_SUPPORTED, [e])
    refused(capi.OB_NOT_SUPPORTED, None, cols=[_col(5, np.arange(100))] * 65)
    refused(capi.OB_INVALID_ARGUMENT, None, rpb=0)
    refused(capi.OB_INVALID_ARGUMENT, None, rk=2)
    refused(capi.OB_INVALID_ARGUMENT, None, align=8)
    refused(capi.OB_INVALID_ARGUMENT, None, align=48)
    # a string obj_type, and bad pointers
    dv = torch.zeros(100, dtype=torch.int64, device="cuda")
    for obj_type, ptr, code in ((capi.OBJ_VARCHAR, dv.data_ptr(), capi.OB_NOT_SUPPORTED), (5, None, capi.OB_INVALID_ARGUMENT)):
        with pytest.raises(capi.ObGpuError) as ei:
            compaction.encode_columns(ctx, [(ptr, None, obj_type, False)], 100, 10, cs=True)
        assert ei.value.code == code
    check(ctx, cols, [INT], 10, 0)[1].free()
    table = writer_table(cols, [INT], 10, 0)
    enc = device_encode(ctx, cols, None, 10, 0)   # encodings None: every column CS_INTEGER
    assert_same_image(enc, table)
    enc.free()


def _largest_rpb(ctx, cols, encs):
    from oceanbase_b200 import capi

    def fits(r):
        try:
            device_encode(ctx, cols, encs, r, 1).free()
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
    """The largest rows_per_block of the cfg5 shape (four integer columns) that fits one CTA, pinned for CS_INTEGER and for
    CS_AUTO (the sort scratch); encoded right there, one row more refused before any launch with the ctx still usable."""
    ctx = _ctx()
    rng = np.random.default_rng(3)
    n = 70_000
    cols = [_col(5, np.arange(n) * 3 + 7), _col(5, rng.integers(0, 1 << 33, n)), _col(5, rng.integers(-(1 << 62), 1 << 62, n)),
            _col(5, rng.integers(0, 1 << 13, n), rng.random(n) < 0.05)]
    got = {}
    for name, encs in (("int", [INT] * 4), ("auto", [AUTO] * 4)):
        lo = _largest_rpb(ctx, cols, encs)
        print(f"largest CS rows_per_block, cfg5 shape, {name}:", lo)
        check(ctx, cols, encs, lo, 1)[1].free()
        got[name] = lo
    assert got == {"int": 6_715, "auto": 2_930}, got
    check(ctx, cols, [AUTO] * 4, 500, 1)[1].free()


def test_launch_count_does_not_depend_on_blocks():
    ctx = _ctx()
    counts = []
    for blocks in (10, 20_000):
        cols = [_col(5, np.arange(blocks * 7)), _col(4, np.arange(blocks * 7) % 5)]
        before = ctx.launch_count
        enc = device_encode(ctx, cols, [INT, AUTO], 7, 1)
        enc.info()
        counts.append(ctx.launch_count - before)
        enc.free()
    assert counts[0] == counts[1] == 1, counts
