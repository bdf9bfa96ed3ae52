"""GROUP BY over a whole scan with one group per distinct value of the page batch (obgpu_result_group_by_values /
obgpu_result_fetch_groups, ScanResult.group_by_values) against a plain value model: the true cells of the selected rows grouped
by value, sorted in the column's own order (signed types signed, unsigned ones unsigned, strings bytewise as unsigned bytes with a
proper prefix first), the NULL group last, each group folded with test_aggregate_exact.fold and encoded as exact_group_by_model
encodes a group. Every comparison is exact.

Cases: 1. every integer type x value codec of the aggregate matrix, every group column (PAX DICT int / DICT string / RLE / CONST,
CS INT_DICT / STR_DICT), five filters, and the same groups merged by value on the host from obgpu_result_group_by +
read_distinct; 2. every count-kernel path of path_table (pipelined kernels on and off, skip index on and off, a
capacity-overflowed scan); 3. one value under different dictionary layouts: PAX entry widths, CS bases under three stream codecs,
PAX and CS blocks in one batch, an all-NULL CS block and const-encoded refs; 4. strings whose hash tags collide, the empty string
next to NULL, NUL bytes and bytes >= 0x80, also from LZ4-stored blocks whose bytes exist only in the device image; 5. the
65 536-value cap; 6. refusals and bad arguments; 7. both fold paths -- CTA-private shared accumulators when
(n_keys + 1) x (n_aggs + 1) x 16 bytes fits gvals::kSharedAccBudget (48 KiB), global ones otherwise (the cap table) -- a
dictionary too large for a warp's rank array, and 128-bit carries over more than 4 M rows; 8. rows selected by a column-group
bitmap; 9. the bench's cfg3 segment against the numpy rebuild of its seeds."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import (COUNT, MAX, MIN, SUM, SUM_PRODUCT, K, M, MATRIX, VB, fold, matrix_spec, matrix_table,
                                  oracle_value, to_i64)
from test_gpu_aggregate_exact import GROUP_AGGS, PATH_AGGS, PATH_ROWS, path_table
from test_scan_codes_model import (CAP, CS_MODES, TYPE_IDS, auto_table, bench_model, bench_string, bench_workload, cap_table,
                                   concat_table, cs_table, cs_uncodable_table, int_layout_table, string_table)

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
UNSIGNED = {6, 7, 8, 9, 10, 21}
OBJ_INT, OBJ_UINT64, OBJ_VARCHAR = 5, 10, 22


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def encode(kind, col, members, cells):
    """one group's aggregate as the device encodes it (exact_group_by_model's encoding)"""
    if kind == COUNT and col < 0:
        return (len(members), 0)
    got = fold(kind, [cells[col][r] for r in members])
    if kind == COUNT:
        return (got, 0)
    if kind == SUM:
        return (to_i64(got), to_i64(got >> 64))
    return (0, 0) if got is None else (to_i64(got), 1)


def value_model(gcells, rows, aggs, cells):
    """(keys, out): the groups of the rows by the value gcells[row], ascending, the NULL group (None) last"""
    groups = {}
    for r in rows:
        groups.setdefault(gcells[r], []).append(r)
    keys = sorted(k for k in groups if k is not None) + ([None] if None in groups else [])
    out = np.zeros((len(aggs), len(keys), 2), dtype=np.int64)
    for g, key in enumerate(keys):
        for k, (kind, col) in enumerate(aggs):
            out[k, g] = encode(kind, col, groups[key], cells)
    return keys, out


def assert_groups(res, gc, aggs, gcells, rows, cells, what):
    got_keys, got = res.group_by_values(gc, aggs)
    want_keys, want = value_model(gcells, rows, aggs, cells)
    assert got_keys == want_keys, what
    assert np.array_equal(got, want), what
    return got_keys, got


def host_merge(batch, res, gc, aggs, gtype, agg_types, image):
    """the second device path: obgpu_result_group_by's per-(block, entry) groups merged by value on the host through
    read_distinct (aggs[0] must be COUNT(*): it tells the empty groups)"""
    goff, out = res.group_by(gc, aggs)
    acc = {}
    for b in range(batch.n_blocks):
        vals, lens = batch.read_distinct(b, gc)
        n = len(vals)
        for g in range(n + 1):
            j = goff[b] + g
            if out[0, j, 0] == 0:
                continue
            if g == n:
                key = None
            elif gtype == OBJ_VARCHAR:
                key = bytes(image[int(vals[g]):int(vals[g]) + int(lens[g])])
            else:
                key = oracle_value(gtype, int(vals[g]))
            st = acc.setdefault(key, [None] * len(aggs))
            for k, (kind, c) in enumerate(aggs):
                lo, hi = int(out[k, j, 0]), int(out[k, j, 1])
                if kind in (COUNT, SUM):
                    st[k] = (st[k] or 0) + (lo if kind == COUNT else (hi << 64) | (lo & M64))
                elif hi:
                    v = lo & M64 if agg_types[c] in UNSIGNED else lo
                    st[k] = v if st[k] is None else (min if kind == MIN else max)(st[k], v)
    keys = sorted(k for k in acc if k is not None) + ([None] if None in acc else [])
    merged = np.zeros((len(aggs), len(keys), 2), dtype=np.int64)
    for g, key in enumerate(keys):
        for k, (kind, _) in enumerate(aggs):
            v = acc[key][k]
            if kind == COUNT:
                merged[k, g] = (v, 0)
            elif kind == SUM:
                merged[k, g] = (to_i64(v), to_i64(v >> 64))
            elif v is not None:
                merged[k, g] = (to_i64(v), 1)
    return keys, merged


# ---- 1. every type x codec x group column -----------------------------------------------------------------------------------
@pytest.mark.parametrize("tname,codec", MATRIX)
def test_matrix(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    table = matrix_table(tname, codec)
    batch = ctx.open_batch(table)
    n, m, vb = spec.n, spec.truth[M], spec.truth[VB]
    cases = [("no filter", None, range(n)), ("every row", ob.White(K, ob.WHITE_OP_GE, (0,)), range(n)),
             ("M < 40", ob.White(M, ob.WHITE_OP_LT, (40,)), [i for i in range(n) if m[i] < 40]),
             ("no row", ob.White(K, ob.WHITE_OP_LT, (0,)), []),
             ("VB NULL", ob.White(VB, ob.WHITE_OP_NU, ()), [i for i in range(n) if vb[i] is None])]
    image = np.asarray(table.image)
    for gname, gc in spec.group_cols.items():
        for what, flt, rows in cases:
            res = batch.scan(flt, [K])
            keys, got = assert_groups(res, gc, GROUP_AGGS, spec.truth[gc], list(rows), spec.truth, (gname, what))
            if what == "no row":
                assert keys == [] and got.shape == (len(GROUP_AGGS), 0, 2)
            if what in ("no filter", "M < 40"):
                hk, hout = host_merge(batch, res, gc, GROUP_AGGS, spec.obj_types[gc], spec.obj_types, image)
                assert hk == keys and np.array_equal(hout, got), (gname, what)
            res.free()
    batch.close()


# ---- 2. every count-kernel path ---------------------------------------------------------------------------------------------
_path_cells = {}


def path_cells(ob, rpb):
    """path_table's truth with its group columns (2 INT DICT, 3 VARCHAR DICT, 4 INT RLE) read back through the oracle"""
    if rpb not in _path_cells:
        table, agg, truth, blocks = path_table(ob, rpb)
        cells = list(truth)
        for c in (2, 3, 4):
            cells[c] = [oracle_value(OBJ_VARCHAR if c == 3 else OBJ_INT, blk.cell(c, r)) for blk in blocks for r in range(blk.row_count)]
        _path_cells[rpb] = cells
    return _path_cells[rpb]


@pytest.fixture(params=["1", "0"], ids=["pipe", "no_pipe"])
def pipe(request, monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", request.param)
    return request.param


@pytest.mark.parametrize("rpb", [1, 133, 1100, 2000])
def test_every_count_path(ob, ctx, pipe, rpb):
    table, agg, truth, blocks = path_table(ob, rpb)
    cells = path_cells(ob, rpb)
    n = PATH_ROWS[rpb]
    m = truth[M]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    cases = [("no filter", None, lambda i: True), ("every row", ob.White(0, ob.WHITE_OP_GE, (0,)), lambda i: True),
             ("key range", ob.White(0, ob.WHITE_OP_BT, (lo, hi)), lambda i: lo <= i <= hi),
             ("key range and m", ob.And([ob.White(0, ob.WHITE_OP_BT, (lo, hi)), ob.White(1, ob.WHITE_OP_LT, (50,))]),
              lambda i: lo <= i <= hi and m[i] < 50)]
    batch = ctx.open_batch(table)
    for with_index in (False, True):
        batch.set_agg_rows(*agg) if with_index else batch.set_agg_rows(None)
        for what, flt, keep in cases:
            res = batch.scan(flt, [0])
            if with_index and what == "key range":
                never, always = res.skip_info()
                assert never > 0 and always > 0, (never, always)
            rows = [i for i in range(n) if keep(i)]
            capped = batch.scan(flt, [0], max_selected_rows=max(len(rows) // 3, 1)) if len(rows) > 1 else None
            for gc in (2, 3, 4):
                for aggs in PATH_AGGS:
                    keys, got = assert_groups(res, gc, aggs, cells[gc], rows, cells, (what, with_index, gc))
                    if capped is not None:    # the scan overflowed its capacity: its bitmap still selects every row
                        ck, cgot = capped.group_by_values(gc, aggs)
                        assert ck == keys and np.array_equal(cgot, got), (what, with_index, gc)
            if capped is not None:
                capped.free()
            res.free()
    batch.close()


# ---- 3. canonical keys across layouts and formats ------------------------------------------------------------------------------
def check_table(ctx, t, group_cols, aggs, image=None, **kw):
    batch = ctx.open_batch(t.image if image is None else image, **kw)
    half = t.n // 2
    import oceanbase_b200 as ob
    for flt, rows in ((None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half])):
        res = batch.scan(flt, [0])
        for gc in group_cols:
            assert_groups(res, gc, aggs, t.cells[gc], list(rows), t.cells, (t.name, gc, flt is None))
        res.free()
    batch.close()


@pytest.mark.parametrize("tname", TYPE_IDS)
@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
def test_int_layouts(ctx, tname, byte_packing):
    t = int_layout_table(tname, byte_packing)
    aggs = [(COUNT, -1), (COUNT, 1), (SUM, 0), (MIN, 0), (MAX, 0), (SUM, 1), (MIN, 1), (MAX, 1)]
    check_table(ctx, t, [1], aggs)


@pytest.mark.parametrize("mode", CS_MODES)
def test_cs_dictionaries(ctx, mode):
    aggs = [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (SUM, 3), (MIN, 2)]
    check_table(ctx, cs_table(mode), [1, 2, 3, 4], aggs)


def test_pax_and_cs_in_one_batch(ctx):
    t = concat_table()
    assert t.image.n_blocks > 12
    check_table(ctx, t, [1, 2, 3, 4], [(COUNT, -1), (SUM, 1), (MIN, 2), (MAX, 3), (COUNT, 1)])


def test_cs_all_null_block_and_const_refs(ctx):
    t = cs_uncodable_table()
    check_table(ctx, t, [1, 2, 3], [(COUNT, -1), (COUNT, 1), (SUM, 2), (MIN, 3), (MAX, 1)])


# ---- 4. strings -------------------------------------------------------------------------------------------------------------
STR_AGGS = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 4), (COUNT, 4)]


def test_strings(ctx):
    t = string_table()
    check_table(ctx, t, [1, 2], STR_AGGS)
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    keys, _ = res.group_by_values(2, STR_AGGS)
    assert b"" in keys and keys[-1] is None and keys.index(b"a\x7fb") < keys.index(b"a\x80b") < keys.index(b"a\xffb")
    assert keys.index(b"a\x00b") < keys.index(b"ab") < keys.index(b"a\x7fb")      # 0x00 < 0x62 < 0x7f, unsigned
    keys1, _ = res.group_by_values(1, STR_AGGS)
    assert len(keys1) == t.distinct(1) + (None in t.cells[1])
    res.free()
    batch.close()


def test_strings_from_stored_blocks(ob, ctx):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    comp = ob.capi.COMPRESSOR_LZ4
    check_table(ctx, t, [1, 2], STR_AGGS, image=compress_table(t.image, comp), compressor=comp)


# ---- 5. the cap -------------------------------------------------------------------------------------------------------------
def test_cap(ob, ctx):
    t = cap_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0), (MAX, 0)]
    keys, _ = assert_groups(res, 1, aggs, t.cells[1], range(t.n), t.cells, "65536 values")
    assert len(keys) == CAP
    with pytest.raises(ob.ObGpuError) as e:
        res.group_by_values(2, aggs)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    assert_groups(res, 1, aggs, t.cells[1], range(t.n), t.cells, "65536 values again")
    res.free()
    batch.close()


# ---- 6. refusals and arguments ----------------------------------------------------------------------------------------------
def test_refusals_and_arguments(ob, ctx):
    lib = ob.capi.lib
    a = auto_table()
    batch = ctx.open_batch(a.image)
    res = batch.scan(None, [0])
    ng, kb, hn = C.c_int64(), C.c_int64(), C.c_int32()
    keys, out = np.zeros(8, dtype=np.int64), np.zeros(64, dtype=np.int64)
    # a fetch before any group-by on this result
    assert lib.obgpu_result_fetch_groups(res._h, keys.ctypes.data, None, out.ctypes.data) == ob.OB_INVALID_ARGUMENT

    def call(gc, aggs):
        spec = np.array(aggs, dtype=np.int32).reshape(-1, 2)
        return lib.obgpu_result_group_by_values(res._h, gc, spec.ctypes.data if len(aggs) else None, len(aggs), C.byref(ng), C.byref(kb),
                                                C.byref(hn))

    for gc in (1, 2):     # OBGPU_ENC_AUTO columns with RAW blocks
        assert call(gc, [(COUNT, -1)]) == ob.OB_NOT_SUPPORTED, gc
    assert call(3, []) == ob.OB_INVALID_ARGUMENT
    assert call(3, [(COUNT, -1)] * 17) == ob.OB_INVALID_ARGUMENT
    assert call(3, [(SUM_PRODUCT, 1)]) == ob.OB_NOT_SUPPORTED
    assert call(3, [(SUM, 2)]) == ob.OB_NOT_SUPPORTED        # a string aggregate column
    assert call(4, [(COUNT, -1)]) == ob.OB_INVALID_ARGUMENT
    assert call(-1, [(COUNT, -1)]) == ob.OB_INVALID_ARGUMENT
    # a refused call leaves no groups behind; the ctx still works
    assert lib.obgpu_result_fetch_groups(res._h, keys.ctypes.data, None, out.ctypes.data) == ob.OB_INVALID_ARGUMENT
    assert_groups(res, 3, [(COUNT, -1)] * 16, a.cells[3], range(a.n), a.cells, "16 aggregates")
    res.free()
    batch.close()


# ---- 7. both fold paths, the per-row probe, 128-bit carries over more than 4 M rows -----------------------------------------
def test_fold_paths(ob, ctx):
    # 16 groups, every aggregate: shared accumulators; cap_table column 1 (test_cap): global ones
    table, agg, truth, blocks = path_table(ob, 2000)
    cells = path_cells(ob, 2000)
    batch = ctx.open_batch(table)
    res = batch.scan(None, [0])
    aggs = PATH_AGGS[0] + PATH_AGGS[1][1:]
    for part in (aggs[:16], aggs[16:]):
        keys, _ = assert_groups(res, 2, part, cells[2], range(PATH_ROWS[2000]), cells, "16 groups")
        assert len(keys) == 17
    res.free()
    batch.close()
    # dictionaries of ~860 entries per block: more than a warp's rank array, ranks probed per row
    rng = np.random.default_rng(5)
    n = 8000
    v = rng.integers(0, 1000, n).astype(np.int64) * 3 - 1500
    w = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    cols = [ob.Column(OBJ_INT, ob.ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(OBJ_INT, ob.ENC_DICT, v), ob.Column(OBJ_INT, ob.ENC_RAW, w)]
    t = ob.encode_table(cols, 2000)
    assert ora.Block(t.block(0)).dict_count(1) > 256
    c = [list(range(n)), v.tolist(), w.tolist()]
    batch = ctx.open_batch(t)
    res = batch.scan(ob.White(0, ob.WHITE_OP_LT, (5000,)), [0])
    assert_groups(res, 1, [(COUNT, -1), (SUM, 2), (MIN, 2), (MAX, 2)], c[1], range(5000), c, "large dictionaries")
    res.free()
    batch.close()


def test_carries_over_four_million_rows(ob, ctx):
    n = (1 << 22) + 12_345
    rng = np.random.default_rng(78)
    g = rng.integers(0, 5, n).astype(np.int64) * 1000 - 2000
    a = rng.integers(1 << 62, (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)    # INT near INT64_MAX
    a[rng.random(n) < 0.02] = np.iinfo(np.int64).min
    u = rng.integers(1 << 63, M64, size=n, dtype=np.uint64, endpoint=True)              # UINT64 near 2^64 - 1
    u[rng.integers(0, n, size=50)] = 0
    m = rng.integers(0, 100, n).astype(np.int64)
    cols = [ob.Column(OBJ_INT, ob.ENC_RAW, m), ob.Column(OBJ_INT, ob.ENC_DICT, g), ob.Column(OBJ_INT, ob.ENC_RAW, a),
            ob.Column(OBJ_UINT64, ob.ENC_RAW, u.view(np.int64))]
    t = ob.encode_table(cols, 2000)
    aggs = [(COUNT, -1), (SUM, 2), (SUM, 3), (MIN, 3), (MAX, 3), (MIN, 2), (MAX, 2)]
    batch = ctx.open_batch(t)
    for flt, sel in ((None, np.ones(n, dtype=bool)), (ob.White(0, ob.WHITE_OP_LT, (50,)), m < 50)):
        res = batch.scan(flt, [0])
        keys, got = res.group_by_values(1, aggs)
        gs, as_, us = g[sel], a[sel], u[sel]
        assert keys == sorted(set(gs.tolist()))
        for j, key in enumerate(keys):
            mask = gs == key
            av, uv = [int(x) for x in as_[mask].tolist()], [int(x) for x in us[mask].tolist()]
            assert sum(av) >= 1 << 64 and sum(uv) >= 1 << 64
            want = [(len(av), 0)] + [encode(kind, 0, range(len(x)), [x]) for kind, x in
                                     ((SUM, av), (SUM, uv), (MIN, uv), (MAX, uv), (MIN, av), (MAX, av))]
            assert [tuple(int(z) for z in got[k, j]) for k in range(len(aggs))] == want, (key, flt is None)
        res.free()
    batch.close()


# ---- 8. rows selected by a column-group bitmap ------------------------------------------------------------------------------
def test_bitmap_selected_rows(ob, ctx):
    table, agg, truth, blocks = path_table(ob, 133)
    cells = path_cells(ob, 133)
    n = PATH_ROWS[133]
    other = ctx.open_batch(table)
    sel = other.scan(ob.White(1, ob.WHITE_OP_LT, (30,)), [0])
    bm = ob.CGBitmap(ctx, n)
    bm.apply(sel, 0, "set")
    batch = ctx.open_batch(table)
    res = batch.scan_bitmap(bm, [0])
    rows = [i for i in range(n) if truth[M][i] < 30]
    for gc in (2, 3, 4):
        assert_groups(res, gc, PATH_AGGS[1], cells[gc], rows, cells, ("bitmap", gc))
    res.free()
    batch.close()
    sel.free()
    other.close()
    bm.free()


# ---- 9. the bench's cfg3 segment ----------------------------------------------------------------------------------------------
def test_bench_segment(ctx):
    w = bench_workload()
    ints, strs = bench_model()
    n = w.table.total_rows
    c0 = ints[0][0][ints[0][1][:n]].tolist()
    c1 = ints[1][0][ints[1][1][:n]].tolist()
    c8 = [bench_string(strs, 8, int(k)) for k in strs[8][1][:n].tolist()]
    cells = {0: c0, 1: c1, 8: c8}
    batch = ctx.open_batch(w.table)
    res = batch.scan(None, [0])
    aggs = [(COUNT, -1), (SUM, 1), (MIN, 1), (MAX, 1)]
    for gc in (0, 8):
        keys, _ = assert_groups(res, gc, aggs, cells[gc], range(n), cells, ("cfg3", gc))
        assert len(keys) == len(set(cells[gc]))
    res.free()
    batch.close()
