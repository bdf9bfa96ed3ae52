"""Skip-index aggregate rows built on the device (obgpu_agg_rows / obgpu_merge_result_agg_rows): rows and offsets byte for byte
what the host writer's obgpu_writer_table_agg_rows builds over the same rows, for every integer class, boundary images, NULL /
NOP patterns and blockings; over merge results; attached to a device-encoded page batch they prune scans like the writer's
rows; and every refused argument leaves the context usable."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# every OBGPU_OBJ_* of an integer class: TINYINT .. UINT64, DATETIME, TIMESTAMP, DATE, TIME, YEAR
INT_TYPES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 17, 18, 19, 20, 21]
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def upload(cols):
    """cols: (obj_type, int64 values, NULL bytes or None) -> (encode_columns tuples, tensors to keep alive)."""
    import torch
    keep, out = [], []
    for t, v, nl in cols:
        dv = torch.from_numpy(np.ascontiguousarray(v, dtype=np.int64)).cuda()
        dn = torch.from_numpy(np.ascontiguousarray(nl, dtype=np.uint8)).cuda() if nl is not None else None
        keep += [dv, dn]
        out.append((dv.data_ptr(), dn.data_ptr() if dn is not None else None, t, False))
    return out, keep


def writer_rows(ob, cols, agg, rpb):
    return ob.table_agg_rows([ob.Column(t, ob.ENC_RAW, np.asarray(v, dtype=np.int64), nulls=nl) for t, v, nl in cols], agg, rpb)


def device_rows(ctx, cols, agg, rpb):
    from oceanbase_b200 import compaction
    dcols, keep = upload(cols)
    return compaction.agg_rows(ctx, dcols, agg, len(cols[0][1]), rpb)


def check(ob, ctx, cols, agg, rpb):
    want_rows, want_off = writer_rows(ob, cols, agg, rpb)
    rows, off = device_rows(ctx, cols, agg, rpb)
    assert np.array_equal(off, want_off), np.nonzero(off != want_off)[0][:5]
    assert np.array_equal(rows, want_rows), int(np.nonzero(rows != want_rows)[0][0]) if rows.size == want_rows.size else (rows.size, want_rows.size)
    return rows, off


def boundary_values(rng, t, n):
    """Random images with the boundaries of every width: INT64_MIN / MAX, UINT64_MAX (-1), above 2^63, and 32-bit values
    whose bits above the datum differ (the compare image takes the low datum_len bytes only)."""
    v = rng.integers(I64_MIN, I64_MAX, size=n, dtype=np.int64, endpoint=True)
    edges = np.array([I64_MIN, I64_MAX, -1, 0, 1, (1 << 63) + 5 - (1 << 64), 0x7FFFFFFF, -0x80000000, 0xFFFFFFFF,
                      (0x1234 << 32) | 0x80000000, (0x5678 << 32) | 0x7FFFFFFF, 0xFF, 0x7F, 0x80], dtype=object)
    edges = np.array([int(e) - (1 << 64) if int(e) > I64_MAX else int(e) for e in edges], dtype=np.int64)
    v[rng.choice(n, size=min(n, 3 * edges.size), replace=False)] = np.tile(edges, 3)[:min(n, 3 * edges.size)]
    small = rng.random(n) < 0.3
    v[small] = rng.integers(-300, 300, size=int(small.sum()))
    return v


def null_bytes(rng, n, rpb, p=0.1):
    nl = (rng.random(n) < p).astype(np.uint8)
    nl[:rpb] = 1                                         # block 0: every cell NULL
    nl[rpb:2 * rpb] = 0                                  # block 1: no NULL
    nl[2 * rpb + 3] = 2                                  # block 2: a NOP cell (the column is not aggregated there)
    return nl


@pytest.mark.parametrize("obj_type", INT_TYPES)
def test_every_integer_class_equals_the_writer(ob, ctx, obj_type):
    rng = np.random.default_rng(obj_type)
    n, rpb = 3001, 37                                    # ragged last block
    cols = [(obj_type, boundary_values(rng, obj_type, n), null_bytes(rng, n, rpb)),
            (obj_type, boundary_values(rng, obj_type, n), None),                         # no NULL pointer
            (obj_type, rng.integers(0, 3, size=n), (rng.random(n) < 0.5).astype(np.uint8))]
    rows, off = check(ob, ctx, cols, [0, 1, 2], rpb)
    assert off.size == (n + rpb - 1) // rpb + 1


@pytest.mark.parametrize("rpb", [1, 133, 1000, 1005])
def test_blockings(ob, ctx, rpb):
    """rows_per_block 1, a ragged one, equal to the row count and larger than it."""
    rng = np.random.default_rng(rpb)
    n = 1000
    cols = [(5, np.sort(rng.integers(-1000, 1000, n)), None), (10, boundary_values(rng, 10, n), (rng.random(n) < 0.2).astype(np.uint8)),
            (19, boundary_values(rng, 19, n), (rng.random(n) < 0.01).astype(np.uint8) * 2)]
    check(ob, ctx, cols, [0, 1, 2], rpb)


def test_unsorted_strict_subset(ob, ctx):
    rng = np.random.default_rng(3)
    n, rpb = 5000, 256
    cols = [(t, boundary_values(rng, t, n), null_bytes(rng, n, rpb) if i % 2 else None) for i, t in enumerate([5, 1, 10, 21, 4, 9])]
    check(ob, ctx, cols, [4, 0, 3, 1], rpb)
    check(ob, ctx, cols, [5, 2], rpb)


def test_wide_index_sizes(ob, ctx):
    """Column indexes >= 256 (idx_size 2) and rows above 255 bytes (idx_off_size 2)."""
    rng = np.random.default_rng(4)
    n, rpb = 2000, 100
    v = boundary_values(rng, 5, n)
    nl = null_bytes(rng, n, rpb)
    cols = [(5, v, nl)] * 300
    rows, off = check(ob, ctx, cols, [299, 256, 3, 0], rpb)
    assert rows[6] & 0x3F == 2                           # agg_col_idx_size
    rows, off = check(ob, ctx, cols, list(range(40, 0, -3)) + [280], rpb)
    b = int(np.argmax(np.diff(off)))
    assert off[b + 1] - off[b] > 255
    assert ((int(rows[off[b] + 6]) | int(rows[off[b] + 7]) << 8) >> 6) & 0x7 == 2   # agg_col_idx_off_size


def test_launch_count_does_not_depend_on_the_block_count(ob, ctx):
    rng = np.random.default_rng(5)
    counts = []
    for n, rpb in ((60_000, 3), (60_000, 6000)):          # 20 000 blocks and 10
        cols = [(5, boundary_values(rng, 5, n), (rng.random(n) < 0.1).astype(np.uint8)), (9, rng.integers(0, 1 << 32, n), None)]
        before = ctx.launch_count
        rows, off = device_rows(ctx, cols, [1, 0], rpb)
        counts.append(ctx.launch_count - before)
        want = writer_rows(ob, cols, [1, 0], rpb)
        assert off.size == n // rpb + 1
        assert np.array_equal(off, want[1]) and np.array_equal(rows, want[0])
    assert counts[0] == counts[1], counts


def _runs(ob, rng, composite, n_runs=3, n=4000):
    tables = []
    for r in range(n_runs):
        key = np.sort(rng.choice(12_000, size=n, replace=False)).astype(np.int64)
        cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, key)]
        if composite:
            cols.append(ob.Column(ob.OBJ_INT, ob.ENC_RAW, (key % 3).astype(np.int64)))
        flag = np.where(rng.random(n) < 0.08, ob.DF_DELETE, ob.DF_INSERT if r == 0 else ob.DF_UPDATE).astype(np.int64)
        cols += [ob.Column(ob.OBJ_TINYINT, ob.ENC_RAW, flag),
                 ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(-1 << 40, 1 << 40, n), nulls=(rng.random(n) < 0.15).astype(np.uint8)),
                 ob.Column(ob.OBJ_UINT64, ob.ENC_RAW, boundary_values(rng, 10, n)),
                 ob.Column(ob.OBJ_INT, ob.ENC_RAW, np.zeros(n, dtype=np.int64), nulls=np.ones(n, dtype=np.uint8))]   # all NULL
        tables.append(ob.encode_table(cols, 500, rowkey_cnt=2 if composite else 1))
    return tables


@pytest.mark.parametrize("composite", [False, True])
def test_merge_result_equals_the_writer_over_fetched_rows(ob, ctx, composite):
    from oceanbase_b200 import compaction
    rng = np.random.default_rng(6 + composite)
    batches = [ob.PageBatch(ctx, t) for t in _runs(ob, rng, composite)]
    base = 2 if composite else 1
    res = compaction.merge_batches(ctx, batches, [0, 1] if composite else 0, base, [base + 1, base + 2, base + 3])
    assert res.info().dropped_deletes > 0
    group = [-1] + ([-2] if composite else []) + [0, 1, 2]
    types = [ob.OBJ_INT] * (len(group) - 2) + [ob.OBJ_UINT64, ob.OBJ_INT]
    host = []
    for c, t in zip(group, types):
        v, nl = res.fetch(c)
        host.append((t, v, nl if c >= 0 else None))
    assert host[-1][2].all()
    for agg, rpb in ((list(range(len(group))), 700), ([len(group) - 2, 0, len(group) - 3], 129)):
        rows, off = res.agg_rows(group, types, agg, rpb)
        want = writer_rows(ob, host, agg, rpb)
        assert np.array_equal(off, want[1]) and np.array_equal(rows, want[0]), (agg, rpb)
    res.free()
    for b in batches:
        b.close()


def test_closed_loop_on_the_device(ob, ctx):
    """Encode with AUTO, open the device image as a page batch, attach the device-built rows: verdicts equal those of the
    writer's rows, a pruned scan returns the unpruned scan's rows, and a range on the sorted rowkey really skips blocks."""
    from oceanbase_b200 import capi, compaction
    from oceanbase_b200.sstable import TableImage
    rng = np.random.default_rng(7)
    n, rpb = 30_000, 700
    cols = [(5, np.arange(n, dtype=np.int64) * 3 - 20_000, None),
            (5, rng.integers(-50, 50, n), (rng.random(n) < 0.05).astype(np.uint8)),
            (10, np.sort(boundary_values(rng, 10, n).view(np.uint64)).view(np.int64), None),
            (19, np.sort(rng.integers(8000, 9500, n)), None)]
    dcols, keep = upload(cols)
    enc = compaction.encode_columns(ctx, dcols, n, rpb, rowkey_cnt=1, keep=keep, encodings=[capi.ENC_AUTO] * 4)
    img, off, sz = enc.fetch()
    assert (sz > 0).all()
    d_img, _, _ = enc.device_image()
    batch = ob.PageBatch(ctx, TableImage(img, off, sz, n, 4), device_image_ptr=d_img, image_size=img.size)
    rows, roff = compaction.agg_rows(ctx, dcols, [0, 1, 2, 3], n, rpb)
    want = writer_rows(ob, cols, [0, 1, 2, 3], rpb)
    assert np.array_equal(rows, want[0]) and np.array_equal(roff, want[1])
    W = ob.White
    flts = [W(0, ob.WHITE_OP_BT, (10_000, 25_000)), W(0, ob.WHITE_OP_LT, (-15_000,)), W(1, ob.WHITE_OP_NU, ()),
            W(1, ob.WHITE_OP_GT, (40,)), W(3, ob.WHITE_OP_GE, (9300,)), W(2, ob.WHITE_OP_LT, (int(cols[2][1][3000]),)),
            ob.And([W(0, ob.WHITE_OP_GE, (0,)), W(1, ob.WHITE_OP_NN, ())])]
    plain = {}
    for i, f in enumerate(flts):
        r = batch.scan(f, [0, 1])
        plain[i] = (r.selected_rows, [r.fetch_col(c) for c in range(2)])
        r.free()
    batch.set_agg_rows(*want)
    writer_verdicts = [batch.skip_index_filter(f) for f in flts]
    batch.set_agg_rows(rows, roff)
    for i, f in enumerate(flts):
        assert np.array_equal(batch.skip_index_filter(f), writer_verdicts[i]), i
        r = batch.scan(f, [0, 1])
        assert r.selected_rows == plain[i][0], i
        for c in range(2):
            got, want_c = r.fetch_col(c), plain[i][1][c]
            assert np.array_equal(got[0], want_c[0]) and np.array_equal(got[2], want_c[2]), (i, c)
        if i == 0:
            always_false, _ = r.skip_info()
            assert always_false > 10, always_false
        r.free()
    batch.close()
    enc.free()


def _raw(ob, ctx, dcols, agg, total, rpb, out=None, cap=0, offs=None):
    from oceanbase_b200 import compaction
    arr = compaction._encode_cols(dcols)
    ac = np.ascontiguousarray(agg, dtype=np.int32)
    size = C.c_int64(-7)
    code = ob.lib.obgpu_agg_rows(ctx._h, arr, len(dcols), ac.ctypes.data if ac.size else None, len(ac), total, rpb, out, cap, offs,
                                 C.byref(size))
    return code, size.value


def _writer_code(ob, cols, agg, total, rpb):
    from oceanbase_b200 import sstable
    arr = sstable._inputs([ob.Column(t, ob.ENC_RAW, np.asarray(v, dtype=np.int64), nulls=nl) for t, v, nl in cols])
    ac = np.ascontiguousarray(agg, dtype=np.int32)
    size = C.c_int64(0)
    return sstable.lib.obgpu_writer_table_agg_rows(arr, len(cols), ac.ctypes.data if ac.size else None, len(ac), total, rpb, None, 0,
                                                   None, C.byref(size))


def test_errors_leave_the_context_usable(ob, ctx):
    rng = np.random.default_rng(8)
    n = 500
    cols = [(5, rng.integers(-9, 9, n), None), (9, rng.integers(0, 9, n), (rng.random(n) < 0.2).astype(np.uint8))]
    dcols, keep = upload(cols)
    inval, unsup, short = ob.OB_INVALID_ARGUMENT, ob.OB_NOT_SUPPORTED, ob.OB_BUF_NOT_ENOUGH
    before = ctx.launch_count
    for agg, rpb, want in (([], 100, inval), ([2], 100, inval), ([-1], 100, inval), ([0, 1, 0], 100, inval), ([0], 0, inval),
                           ([0], -5, inval)):
        assert _raw(ob, ctx, dcols, agg, n, rpb)[0] == want, (agg, rpb)
        if agg != [0, 1, 0]:                             # the writer merges a repeated column into one cell; the device refuses it
            assert _writer_code(ob, cols, agg, n, rpb) == want, (agg, rpb)
    assert ob.lib.obgpu_agg_rows(ctx._h, None, 2, None, 1, n, 100, None, 0, None, None) == inval
    # a class the device does not aggregate (ObNullType here; strings are the host writer's)
    bad = [(0, cols[0][1], None)] + cols[1:]
    bad_dev, bad_keep = upload(bad)
    assert _raw(ob, ctx, bad_dev, [1, 0], n, 100)[0] == unsup
    assert _writer_code(ob, bad, [1, 0], n, 100) == unsup
    str_dev = [(dcols[0][0], None, ob.OBJ_VARCHAR, False)] + dcols[1:]
    assert _raw(ob, ctx, str_dev, [0], n, 100)[0] == unsup
    assert ctx.launch_count == before                    # every argument error comes before any launch
    # a row above 65535 bytes: 2 200 aggregated 8-byte columns without NULLs (~74 KB per row)
    wide = [(5, cols[0][1], None)] * 2200
    wide_dev = [dcols[0]] * 2200
    assert _writer_code(ob, wide, list(range(2200)), n, 250) == unsup
    assert _raw(ob, ctx, wide_dev, list(range(2200)), n, 250)[0] == unsup
    # out_cap too small: nothing written
    code, size = _raw(ob, ctx, dcols, [0, 1], n, 100)
    assert code == ob.OB_SUCCESS and size > 0
    out = np.full(size, 0xA5, dtype=np.uint8)
    offs = np.full(n // 100 + 1, -3, dtype=np.int64)
    assert _raw(ob, ctx, dcols, [0, 1], n, 100, out.ctypes.data, size - 1, offs.ctypes.data)[0] == short
    assert (out == 0xA5).all() and (offs == -3).all()
    assert _raw(ob, ctx, dcols, [0, 1], n, 100, out.ctypes.data, size, None)[0] == inval
    # the context still works
    check(ob, ctx, cols, [1, 0], 100)
