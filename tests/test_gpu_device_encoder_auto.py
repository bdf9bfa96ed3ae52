"""The device encoder with OBGPU_ENC_AUTO columns (obgpu_encode_columns_ex / obgpu_merge_result_encode_ex): per block and per
column the codec the host writer's choose_auto_encoding picks (RAW, DICT, RLE, CONST, INTEGER_BASE_DIFF), and byte for byte
the blocks obgpu_writer_encode_table writes with the same per-column encodings: image, offsets, sizes, column checksums."""
import numpy as np
import pytest

import oracle_binding as ora

pytestmark = pytest.mark.gpu

RAW, AUTO = 0, 32


def _ctx():
    import oceanbase_b200 as ob
    return ob.ScanContext(0)


def writer_table(cols, encs, rpb, rk, align=128):
    from oceanbase_b200.sstable import Column, encode_table
    return encode_table([Column(t, e, v, nulls=nl, byte_packing_only=bo) for (t, v, nl, bo), e in zip(cols, encs)], rpb,
                        rowkey_cnt=rk, align=align)


def device_encode(ctx, cols, encs, rpb, rk, align=128):
    import torch
    from oceanbase_b200 import compaction
    keep, dcols = [], []
    for (t, v, nl, bo) in cols:
        dv = torch.from_numpy(np.ascontiguousarray(v)).cuda()
        dn = torch.from_numpy(np.ascontiguousarray(nl)).cuda() if nl is not None else None
        keep += [dv, dn]
        dcols.append((dv.data_ptr(), dn.data_ptr() if dn is not None else None, t, bo))
    return compaction.encode_columns(ctx, dcols, len(cols[0][1]), rpb, rowkey_cnt=rk, align=align, keep=keep, encodings=encs)


def first_difference(img, want, off, sz):
    bad = int(np.nonzero(img != want)[0][0])
    blk = int(np.searchsorted(off, bad, side="right") - 1)
    return f"first differing byte {bad} (block {blk}, byte {bad - off[blk]} of {sz[blk]})"


def assert_same_image(enc, table, host_blocks=()):
    """Blocks of size 0 (left to the host writer) must be exactly `host_blocks`; every other block equals the writer's."""
    img, off, sz = enc.fetch()
    info = enc.info()
    assert info.n_blocks == table.n_blocks
    assert sorted(np.nonzero(sz == 0)[0].tolist()) == sorted(host_blocks)
    assert info.n_host_blocks == len(host_blocks)
    want = np.asarray(table.image)
    if not host_blocks:
        assert np.array_equal(off, np.asarray(table.offsets)), "block offsets differ"
        assert np.array_equal(sz, np.asarray(table.sizes)), "block sizes differ"
        assert img.size == want.size, (img.size, want.size)
        if not np.array_equal(img, want):
            raise AssertionError(first_difference(img, want, off, sz))
        return
    for b in range(table.n_blocks):
        if sz[b] == 0:
            continue
        w = np.asarray(table.block(b))
        assert sz[b] == w.size, (b, sz[b], w.size)
        if not np.array_equal(img[off[b]:off[b] + sz[b]], w):
            raise AssertionError(f"block {b}: " + first_difference(img[off[b]:off[b] + sz[b]], w, np.zeros(1, np.int64), sz[b:b + 1]))


def column_types(table, n_cols):
    """(type_ of every column header of every block, CONST blocks with / without exceptions)."""
    img, off, sz = np.asarray(table.image), np.asarray(table.offsets), np.asarray(table.sizes)
    types, const_exc, const_plain = set(), 0, 0
    for b in range(table.n_blocks):
        for c in range(n_cols):
            h = img[off[b] + 64 + 16 * c: off[b] + 64 + 16 * c + 16]
            types.add(int(h[1]))
            if h[1] == 3:
                meta = off[b] + 64 + 16 * n_cols + int(h[8:12].view(np.uint32)[0])
                if img[meta + 1] > 0:
                    const_exc += 1
                else:
                    const_plain += 1
    return types, const_exc, const_plain


def check(ctx, cols, encs, rpb, rk, align=128, host_blocks=()):
    table = writer_table(cols, encs, rpb, rk, align)
    enc = device_encode(ctx, cols, encs, rpb, rk, align)
    assert_same_image(enc, table, host_blocks)
    img, off, sz = enc.fetch()
    for b in sorted({0, len(off) // 2, len(off) - 1}):
        if sz[b]:
            assert ora.Block(img[off[b]:off[b] + sz[b]].copy()).verify_checksums() == 0, b
    o = ora.oracle()
    got = enc.column_checksums()
    for c, (t, v, nl, _bo) in enumerate(cols):
        dl = 1 if t == 21 else (4 if t == 19 else 8)
        v = np.ascontiguousarray(v)
        assert int(got[c]) == o.ora_column_checksum(v.ctypes.data, nl.ctypes.data if nl is not None else None, len(v), dl), c
    return table, enc


def _col(t, v, nl=None, bo=False):
    return (t, np.asarray(v, dtype=np.int64), None if nl is None else np.asarray(nl, dtype=np.uint8), bo)


def shapes():
    """name -> (cols, rows_per_block, rowkey_cnt); every column AUTO."""
    rng = np.random.default_rng(17)
    n = 6_000
    S = {}
    S["rowkey_timestamp"] = ([_col(5, np.arange(n) * 3 + 1_000_000_007), _col(17, 1_700_000_000_000 + np.cumsum(rng.integers(0, 50, n))),
                              _col(5, rng.integers(0, 1 << 40, n))], 500, 1)
    S["low_cardinality"] = ([_col(5, rng.integers(0, 7, n) * 1_000_003), _col(4, rng.integers(-5, 5, n), rng.random(n) < 0.05),
                             _col(10, rng.choice([3, 1 << 40, 77, 1 << 63], n).astype(np.uint64).view(np.int64))], 500, 0)
    S["short_runs"] = ([_col(5, np.repeat(rng.integers(0, 1 << 30, n // 8 + 1), 8)[:n]),
                        _col(5, np.repeat(rng.integers(0, 3, n // 20 + 1), 20)[:n], np.repeat(rng.random(n // 20 + 1) < 0.1, 20)[:n]),
                        _col(2, np.repeat(rng.integers(-300, 300, n // 50 + 1), 50)[:n])], 400, 0)
    near = np.full(n, 42, dtype=np.int64)
    exc = rng.choice(n, 150, replace=False)
    near[exc] = rng.integers(0, 1 << 20, 150)
    nl = np.zeros(n, np.uint8)
    nl[rng.choice(n, 60, replace=False)] = 1
    S["near_constant"] = ([_col(5, near), _col(5, np.full(n, -7), nl), _col(1, np.full(n, -3)), _col(5, np.full(n, 9), np.ones(n))], 600, 0)
    # CONST ties: two values of equal frequency whose first-occurrence and sorted orders disagree (the larger one first), with
    # NULLs as frequent as each of them and without; the two tie-breaks pick different constants and exception rows
    k = 300
    S["const_ties_2"] = ([_col(5, np.tile([9, 3], k)), _col(5, np.tile([5, 5], k), np.tile([1, 0], k)),
                          _col(5, np.tile([8, 8], k), np.tile([0, 1], k)), _col(4, np.tile([200, 7], k))], 2, 0)
    S["const_ties_3"] = ([_col(5, np.tile([9, 3, 0], k), np.tile([0, 0, 1], k)), _col(5, np.tile([9, 9, 3, 3, 4, 4], k // 2)),
                          _col(5, np.tile([0, 7, 7], k), np.tile([1, 0, 0], k))], 3, 0)
    # exceptions before and after the constant, in first-occurrence order unlike the sorted order
    m = 300
    a =np.tile(np.concatenate([np.full(m - 6, 900), [100, 100, 100, 50, 50, 50]]), n // m)
    b = np.tile(np.concatenate([[900, 900, 900], np.full(m - 3, 100)]), n // m)
    tn = np.tile(np.concatenate([np.zeros(m - 3), np.ones(3)]), n // m)
    S["const_ties"] = ([_col(5, a), _col(5, b), _col(5, np.tile(np.concatenate([[5, 5, 5, 8, 8, 8], np.full(m - 6, 6)]), n // m)),
                        _col(5, np.tile(np.concatenate([[8, 8, 8, 5, 5, 5], np.full(m - 6, 6)]), n // m),
                             np.tile(np.concatenate([np.zeros(m - 3), np.ones(3)]), n // m)),
                        _col(5, np.tile(np.concatenate([np.full(m - 6, 6), [8, 8, 8, 5, 5, 5]]), n // m), tn)], m, 0)
    S["narrow_types"] = ([_col(t, rng.integers(lo, hi, n), rng.random(n) < 0.03) for t, lo, hi in
                          ((1, -128, 128), (2, -200, 200), (3, -(1 << 23), 1 << 23), (4, -(1 << 31), 1 << 31), (4, -40, -10),
                           (6, 0, 256), (7, 0, 65536), (8, 0, 1 << 24), (9, 0, 1 << 32), (9, 1000, 1010), (19, 18_000, 18_400),
                           (21, 0, 120))], 500, 0)
    S["negative"] = ([_col(5, -np.arange(n) * 11 - 5), _col(5, rng.integers(-(1 << 62), 1 << 62, n)), _col(5, rng.integers(-20, -10, n)),
                      _col(5, np.repeat(rng.integers(-(1 << 50), -(1 << 49), n // 10 + 1), 10)[:n])], 500, 1)
    S["byte_packing_only"] = ([_col(5, np.arange(n) + 10_000, bo=True), _col(5, rng.integers(0, 9, n), bo=True),
                               _col(5, np.repeat(rng.integers(0, 1 << 33, n // 25 + 1), 25)[:n], rng.random(n) < 0.02, bo=True),
                               _col(4, np.full(n, 3), bo=True), _col(5, rng.integers(0, 1 << 17, n), rng.random(n) < 0.3, bo=True)], 500, 0)
    S["wide"] = ([_col(5, rng.integers(0, k + 2, n) * (k + 1)) for k in range(40)], 300, 0)
    S["tiny_and_ragged"] = ([_col(5, rng.integers(0, 4, 1_003)), _col(5, rng.integers(0, 1 << 40, 1_003), rng.random(1_003) < 0.3)], 1, 0)
    S["ragged"] = ([_col(5, np.arange(2_001) * 2), _col(5, rng.integers(0, 3, 2_001), rng.random(2_001) < 0.1)], 250, 1)
    return S


SHAPES = shapes()


@pytest.mark.parametrize("name", list(SHAPES))
def test_auto_blocks_equal_the_host_writer(name):
    ctx = _ctx()
    cols, rpb, rk = SHAPES[name]
    check(ctx, cols, [AUTO] * len(cols), rpb, rk)[1].free()


def test_every_codec_is_covered():
    """The shapes above make the writer pick all five codecs, and CONST with and without exceptions."""
    types, const_exc, const_plain = set(), 0, 0
    for cols, rpb, rk in SHAPES.values():
        t, ce, cp = column_types(writer_table(cols, [AUTO] * len(cols), rpb, rk), len(cols))
        types |= t
        const_exc += ce
        const_plain += cp
    assert types == {0, 1, 2, 3, 4}, types
    assert const_exc > 0 and const_plain > 0


@pytest.mark.parametrize("align", [16, 128, 4096])
def test_alignments_and_mixed_raw_auto(align):
    ctx = _ctx()
    cols, rpb, rk = SHAPES["low_cardinality"]
    cols = cols + SHAPES["rowkey_timestamp"][0]
    check(ctx, cols, [AUTO, RAW, AUTO, RAW, AUTO, AUTO], rpb, rk, align=align)[1].free()


def test_null_dominated_raw_column_is_left_to_the_host():
    """AUTO keeps RAW on a column of random 64-bit values with half of its cells NULL in one block: the writer estimates the
    var-stored RAW column at 2 bytes a row, below any dictionary, and stores it var-length there. That block reads size 0
    and its neighbours keep the writer's bytes."""
    ctx = _ctx()
    rng = np.random.default_rng(6)
    n, rpb = 4_000, 500
    nl = np.zeros(n, np.uint8)
    nl[1500:2000:2] = 1
    cols = [_col(5, np.arange(n)), _col(5, rng.integers(-(1 << 62), 1 << 62, n), nl), _col(5, rng.integers(0, 4, n))]
    table, enc = check(ctx, cols, [AUTO] * 3, rpb, 1, host_blocks=(3,))
    assert np.asarray(table.block(3))[22] == 1   # opt2_: the writer stored one var column there
    enc.free()


def test_none_is_the_raw_call():
    """encodings=None and all-RAW encodings give today's bytes."""
    ctx = _ctx()
    cols, rpb, rk = SHAPES["negative"]
    table = writer_table(cols, [RAW] * len(cols), rpb, rk)
    for e in (None, [RAW] * len(cols)):
        enc = device_encode(ctx, cols, e, rpb, rk)
        assert_same_image(enc, table)
        enc.free()


def test_shared_memory_limit():
    """The largest rows_per_block that fits, encoded right; one row more is refused before any launch, the ctx still usable."""
    from oceanbase_b200 import capi
    ctx = _ctx()
    rng = np.random.default_rng(3)
    n = 40_000
    cols = [_col(5, np.arange(n) * 3 + 7), _col(5, rng.integers(0, 1 << 33, n)), _col(5, rng.integers(-(1 << 62), 1 << 62, n)),
            _col(5, rng.integers(0, 1 << 13, n), rng.random(n) < 0.05)]   # the cfg5 shape
    encs = [AUTO] * 4

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
    print("largest AUTO rows_per_block, cfg5 shape:", lo)
    check(ctx, cols, encs, lo, 1)[1].free()
    assert not fits(lo + 1)
    check(ctx, cols, encs, 500, 1)[1].free()


def test_other_encodings_are_refused():
    from oceanbase_b200 import capi
    ctx = _ctx()
    cols = [_col(5, np.arange(100))]
    for e in (capi.ENC_DICT, capi.ENC_RLE, capi.ENC_CONST, capi.ENC_INTEGER_BASE_DIFF, capi.ENC_CS_AUTO):
        with pytest.raises(capi.ObGpuError) as ei:
            device_encode(ctx, cols, [e], 10, 0)
        assert ei.value.code == capi.OB_NOT_SUPPORTED
    check(ctx, cols, [AUTO], 10, 0)[1].free()


def test_seeded_random_differential():
    ctx = _ctx()
    rng = np.random.default_rng(2024)
    types = (1, 2, 3, 4, 5, 6, 7, 9, 10, 17, 19, 21)
    for it in range(12):
        n = int(rng.integers(1, 5_000))
        rpb = int(rng.choice([1, 2, 7, 64, 133, 500, 1_000]))
        cols, encs = [], []
        for c in range(int(rng.integers(1, 12))):
            t = int(rng.choice(types))
            kind = int(rng.integers(0, 5))
            if kind == 0:
                v = rng.integers(-(1 << 62), 1 << 62, n)
            elif kind == 1:
                v = rng.integers(-3, 4, n) * int(rng.integers(1, 1 << 20))
            elif kind == 2:
                run = int(rng.integers(1, 40))
                v = np.repeat(rng.integers(-1000, 1000, n // run + 1), run)[:n]
            elif kind == 3:
                v = np.full(n, int(rng.integers(-100, 100)))
                k = int(rng.integers(0, 6))
                v[rng.integers(0, n, k)] = rng.integers(-100, 100, k)
            else:
                v = np.cumsum(rng.integers(0, 1000, n)) - int(rng.integers(0, 1 << 30))
            nf = float(rng.choice([0.0, 0.0, 0.01, 0.2, 0.6]))
            nl = (rng.random(n) < nf) if nf > 0 else None
            cols.append(_col(t, v, nl, bool(rng.random() < 0.2)))
            encs.append(AUTO if rng.random() < 0.8 else RAW)
        table = writer_table(cols, encs, rpb, 0)
        enc = device_encode(ctx, cols, encs, rpb, 0)
        _, _, sz = enc.fetch()
        host = tuple(np.nonzero(sz == 0)[0].tolist())
        for b in host:   # only a block with a RAW column the writer stores var-length may be left to the host
            assert np.asarray(table.block(b))[22] > 0, (it, b)
        assert_same_image(enc, table, host)
        enc.free()


def test_reopen_scan_and_compress():
    """AUTO blocks re-open from the device image as a page batch that scans like the writer's; compressed on the device
    with LZ4 and zstd_1.3.8 they equal the writer's compression of its own image."""
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import TableImage, compress_table
    ctx = _ctx()
    rng = np.random.default_rng(12)
    n = 20_000
    cols = [_col(5, np.arange(n) * 2 + 5), _col(5, rng.integers(0, 40, n), rng.random(n) < 0.07),
            _col(5, np.repeat(rng.integers(0, 1 << 40, n // 30 + 1), 30)[:n]), _col(4, np.full(n, 11))]
    table, enc = check(ctx, cols, [AUTO] * 4, 700, 1)
    img, off, sz = enc.fetch()
    d_img, _, _ = enc.device_image()
    dev = ob.PageBatch(ctx, TableImage(img, off, sz, n, 4), device_image_ptr=d_img, image_size=img.size)
    ref = ob.PageBatch(ctx, table)
    flt = ob.And([ob.White(1, ob.WHITE_OP_LT, [30]), ob.White(0, ob.WHITE_OP_GE, [1000])])
    v1, nl1 = cols[1][1], cols[1][2]
    want = (~nl1.astype(bool)) & (v1 < 30) & (cols[0][1] >= 1000)
    for b in (dev, ref):
        r = b.scan(flt, [0, 2, 3])
        assert r.selected_rows == int(want.sum())
        for i, c in enumerate((0, 2, 3)):
            d, _, _ = r.fetch_col(i)
            assert np.array_equal(d[:r.selected_rows].view(np.int64) if d.dtype.itemsize == 8 else d[:r.selected_rows],
                                  cols[c][1][want] if d.dtype.itemsize == 8 else cols[c][1][want].astype(d.dtype)), c
    dev.close()
    ref.close()
    for comp in (2, 6):
        got = enc.compress(comp)
        g_img, g_off, g_sz = got.fetch()
        st = compress_table(table, comp, align=128)
        assert np.array_equal(g_off, np.asarray(st.offsets)) and np.array_equal(g_sz, np.asarray(st.sizes)), comp
        assert np.array_equal(g_img, np.asarray(st.image)), comp
    enc.free()


def test_column_groups_of_a_merge_result_with_auto():
    """co_merge_write(..., encodings=AUTO): every group equals the host writer with AUTO over the merged rows."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi, compaction
    from oceanbase_b200.sstable import Column, encode_table
    ctx = _ctx()
    rng = np.random.default_rng(9)
    runs = []
    for r in range(3):
        n = 6_000
        key = np.sort(rng.choice(40_000, size=n, replace=False)).astype(np.int64)
        cols = [Column(capi.OBJ_INT, capi.ENC_INTEGER_BASE_DIFF, key),
                Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 5, size=n, dtype=np.int64)),
                Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 1 << 40, size=n, dtype=np.int64), nulls=(rng.random(n) < 0.1).astype(np.uint8)),
                Column(capi.OBJ_INT, capi.ENC_RAW, np.full(n, 77, dtype=np.int64))]
        runs.append(encode_table(cols, 700, rowkey_cnt=1))
    batches = [ob.PageBatch(ctx, t) for t in runs]
    res = compaction.merge_batches(ctx, batches, 0, None, [1, 2, 3])
    key, _ = res.fetch(-1)
    payload = [res.fetch(c) for c in range(3)]
    groups = [[-1, 0, 1, 2], [0], [1], [2, 0]]
    types = {c: capi.OBJ_INT for c in (-1, 0, 1, 2)}
    encs = compaction.co_merge_write(res, groups, types, rows_per_block=900, encodings={c: AUTO for c in (-1, 0, 1, 2)})
    for cg, enc in zip(groups, encs):
        host_cols = []
        for c in cg:
            if c == -1:
                host_cols.append(Column(capi.OBJ_INT, AUTO, key))
            else:
                v, nl = payload[c]
                host_cols.append(Column(capi.OBJ_INT, AUTO, v, nulls=nl if nl.any() else None))
        table = encode_table(host_cols, 900, rowkey_cnt=1 if cg[0] == -1 else 0)
        assert_same_image(enc, table)
        enc.free()
