"""GROUP BY columns of any encoding (obgpu_result_group_by_any, ScanResult.group_by_any) against the plain tuple model of the
generator's cells (test_gpu_group_by_columns.tuple_model), compared exactly: keys, NULLs, string bytes, 128-bit aggregates.

Cases: 1. wherever obgpu_result_group_by_columns accepts a batch, the same fetched bytes and the dictionary path (the aggregate
matrix's group columns under five filters, string, CS and open tables, every count path of path_table with overflowed scans);
2. the cells path over every integer type x codec of the matrix's value columns, key sets mixing dictionary and other columns,
auto_table, every string codec x type x NULL rate, LZ4-, zstd- and zlib-stored batches and a bitmap scan; 3. the limits it
lifts at both sides: the 65 536-value cap, the first capacity 2^20 and its refold (seen in the ctx's launch count), and the
4 194 304-tuple hashed cap of the dictionary fold; 4. one key and sixteen keys over every row with sums past 2^64 and MIN /
MAX at the type extremes; 5. the group slot with obgpu_result_fetch_groups, obgpu_groups_add and the top-rows slot;
6. refusals. test_group_by_any_shapes proves the fixtures' shapes."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM, SUM_PRODUCT, K, M, MATRIX, VA, VB, W, matrix_spec, matrix_table
from test_gpu_aggregate_exact import GROUP_AGGS, PATH_AGGS, PATH_ROWS, path_table
from test_gpu_group_by_columns import np_model, tuple_model
from test_gpu_group_by_values import path_cells
from test_group_by_any_shapes import FIRST_GROUPS, contention_table, refold_table
from test_group_by_columns_shapes import HASH_GROUPS, hash_cap_table
from test_scan_codes_model import CAP, CS_MODES, auto_table, cap_table, cs_table, open_table, string_table
import test_string_filter_exact as sfe

pytestmark = pytest.mark.gpu

DICT, CELLS = 1, 2
STR_AGGS = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 4), (COUNT, 4)]
AUTO_AGGS = [(COUNT, -1), (SUM, 0), (MIN, 3), (MAX, 1), (COUNT, 1)]


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def raw_groups(res, entry, gcols, aggs):
    """the result's groups as obgpu_result_fetch_group_columns returns them, after `entry` (group_by_columns or group_by_any):
    (keys, NULL flags, heap, out) as bytes, and the path (None for group_by_columns); raises on a refusal"""
    from oceanbase_b200 import capi
    lib = capi.lib
    cols = np.array(gcols, dtype=np.int32)
    spec = np.array(aggs, dtype=np.int32).reshape(-1, 2)
    ng, kb, path = C.c_int64(0), C.c_int64(0), C.c_int32(0)
    if entry == "any":
        rc = lib.obgpu_result_group_by_any(res._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb), C.byref(path))
    else:
        rc = lib.obgpu_result_group_by_columns(res._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb))
    if rc != 0:
        return rc, None
    n = ng.value
    keys = np.zeros((len(cols), n + 1), dtype=np.int64)
    nulls = np.zeros((len(cols), max(n, 1)), dtype=np.uint8)
    heap = np.zeros(max(kb.value, 1), dtype=np.uint8)
    out = np.zeros((len(aggs), max(n, 1), 2), dtype=np.int64)
    assert lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data) == 0
    return 0, (keys.tobytes(), nulls.tobytes(), heap[:kb.value].tobytes(), out.tobytes(), path.value if entry == "any" else None)


def assert_same_as_columns(res, gcols, aggs, what):
    """group_by_any where group_by_columns succeeds: the same bytes and the dictionary path; else the cells path. Returns it."""
    rc, cols = raw_groups(res, "columns", gcols, aggs)
    rc_any, anyg = raw_groups(res, "any", gcols, aggs)
    assert rc_any == 0, (what, rc_any)
    if rc == 0:
        assert anyg[:4] == cols[:4] and anyg[4] == DICT, what
    else:
        assert anyg[4] == CELLS, (what, rc)
    return anyg[4]


def assert_any(res, gcols, aggs, cells, rows, what, path=None):
    keys, got, p = res.group_by_any(gcols, aggs)
    want_keys, want = tuple_model([cells[c] for c in gcols], list(rows), aggs, cells)
    assert keys == want_keys, what
    assert np.array_equal(got, want), what
    if path is not None:
        assert p == path, (what, p)
    return keys, got, p


# ---- 1. the dictionary path is untouched ------------------------------------------------------------------------------------
def matrix_filters(ob, spec):
    n, m, vb = spec.n, spec.truth[M], spec.truth[VB]
    return [("no filter", None, range(n)), ("every row", ob.White(K, ob.WHITE_OP_GE, (0,)), range(n)),
            ("M < 40", ob.White(M, ob.WHITE_OP_LT, (40,)), [i for i in range(n) if m[i] < 40]),
            ("no row", ob.White(K, ob.WHITE_OP_LT, (0,)), []),
            ("VB NULL", ob.White(VB, ob.WHITE_OP_NU, ()), [i for i in range(n) if vb[i] is None])]


@pytest.mark.parametrize("tname,codec", MATRIX)
def test_matrix(ob, ctx, tname, codec):
    """dictionary group columns take DICT with group_by_columns' bytes; VA / VB / W / K of every codec match the model, on
    CELLS wherever the column is not dictionary coded; mixed key sets decode dictionary plans on the cells path"""
    spec = matrix_spec(tname, codec)
    batch = ctx.open_batch(matrix_table(tname, codec))
    gcs = list(spec.group_cols.values())
    for what, flt, rows in matrix_filters(ob, spec):
        res = batch.scan(flt, [K])
        for gcols in [[g] for g in gcs] + [list(p) for p in itertools.combinations(gcs, 2)]:
            assert assert_same_as_columns(res, gcols, GROUP_AGGS, (gcols, what)) == DICT
        for gcols in ([VA], [VB], [W], [K], [gcs[-1], VA], [VB, M], [VA, VB, W, K]):
            _, _, p = assert_any(res, gcols, GROUP_AGGS, spec.truth, rows, (gcols, what))
            assert p == assert_same_as_columns(res, gcols, GROUP_AGGS, (gcols, what))
            if codec in ("raw", "raw_bp", "ibd", "cs_integer") and gcols != [K]:
                assert p == CELLS, (gcols, what)
        res.free()
    batch.close()


def check_table(ctx, t, keysets, aggs, image=None, path=None, **kw):
    import oceanbase_b200 as ob
    batch = ctx.open_batch(t.image if image is None else image, **kw)
    half = t.n // 2
    for flt, rows in ((None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half])):
        res = batch.scan(flt, [0])
        for gcols in keysets:
            _, _, p = assert_any(res, gcols, aggs, t.cells, rows, (t.name, gcols, flt is None), path)
            assert p == assert_same_as_columns(res, gcols, aggs, (t.name, gcols))
        res.free()
    batch.close()


def test_dictionary_tables(ctx):
    check_table(ctx, string_table(), [[1, 2], [2, 1], [2, 4, 1]], STR_AGGS, path=DICT)
    check_table(ctx, open_table(), [[1, 3], [3, 2, 1], [2, 1]], [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (SUM, 3)], path=DICT)
    for mode in CS_MODES:
        check_table(ctx, cs_table(mode), [[1, 2], [3, 4], [4, 1, 2]], [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (MIN, 2)])


@pytest.mark.parametrize("rpb", [1, 133, 1100, 2000])
def test_every_count_path(ob, ctx, rpb):
    table, agg, truth, blocks = path_table(ob, rpb)
    cells = path_cells(ob, rpb)
    n = PATH_ROWS[rpb]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    batch = ctx.open_batch(table)
    for flt, keep in ((None, lambda i: True), (ob.White(0, ob.WHITE_OP_BT, (lo, hi)), lambda i: lo <= i <= hi)):
        rows = [i for i in range(n) if keep(i)]
        res = batch.scan(flt, [0])
        capped = batch.scan(flt, [0], max_selected_rows=max(len(rows) // 3, 1))
        for gcols in ([2, 3], [4, 2], [0], [0, 2]):
            for r in (res, capped):   # the capped scan overflowed: its bitmap still selects every row
                keys, got, p = assert_any(r, gcols, PATH_AGGS[1], cells, rows, (rpb, gcols, r is capped))
                assert p == assert_same_as_columns(r, gcols, PATH_AGGS[1], (rpb, gcols))
                if gcols == [0]:
                    assert p == CELLS
        capped.free()
        res.free()
    batch.close()


# ---- 2. every encoding on the cells path ------------------------------------------------------------------------------------
def test_auto_table(ctx):
    check_table(ctx, auto_table(), [[1], [2], [1, 2, 3]], AUTO_AGGS, path=CELLS)


CELLS_CODECS = ("raw_var", "raw_fix", "hex", "string_diff", "string_prefix", "column_equal", "column_substr", "cs_string_var",
                "cs_string_fix")


@pytest.mark.parametrize("codec,tname,nname", sfe.MATRIX, ids=sfe.MATRIX_IDS)
def test_string_codecs(ob, ctx, codec, tname, nname):
    spec = sfe.spec_of(codec, tname, nname)
    batch = ctx.open_batch(sfe.table_of(codec, tname, nname))
    m = spec.truth[1]
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 1), (MAX, 0), (COUNT, 1)]
    for flt, rows in ((None, range(spec.n)), (ob.White(1, ob.WHITE_OP_LT, (30,)), [i for i in range(spec.n) if m[i] < 30])):
        res = batch.scan(flt, [0])
        for gcols in ([2], [2, 3], [1, 2], [3]):
            _, _, p = assert_any(res, gcols, aggs, spec.truth, rows, (gcols, flt is None))
            assert p == assert_same_as_columns(res, gcols, aggs, gcols)
            if gcols == [2]:
                dict_like = spec.s_encoding in (sfe.ENC_DICT, sfe.ENC_CS_STR_DICT, sfe.ENC_RLE, sfe.ENC_CONST)
                assert p == (DICT if dict_like else CELLS), (codec, spec.s_encoding)
                if codec in CELLS_CODECS and spec.s_encoding == sfe.CODECS[codec][0]:
                    assert p == CELLS
        res.free()
    batch.close()


@pytest.mark.parametrize("comp", ["COMPRESSOR_LZ4", "COMPRESSOR_ZSTD_1_3_8", "COMPRESSOR_ZLIB"])
def test_stored_batches(ob, ctx, comp):
    from oceanbase_b200.sstable import compress_table
    c = getattr(ob.capi, comp)
    t = auto_table()
    check_table(ctx, t, [[1], [2, 1]], AUTO_AGGS, image=compress_table(t.image, c), compressor=c, path=CELLS)
    s = string_table()
    check_table(ctx, s, [[1, 2], [0, 2]], STR_AGGS, image=compress_table(s.image, c), compressor=c)


def test_bitmap_scan(ob, ctx):
    t = auto_table()
    batch = ctx.open_batch(t.image)
    flt = ob.White(3, ob.WHITE_OP_LT, (9,))
    rows = [r for r in range(t.n) if t.cells[3][r] < 9]
    sel = batch.scan(flt, [0])
    bm = ob.CGBitmap(ctx, t.n)
    bm.apply(sel, 0, "set")
    other = ctx.open_batch(t.image)
    res = other.scan_bitmap(bm, [0])
    for gcols in ([1], [2, 3]):
        assert_any(res, gcols, AUTO_AGGS, t.cells, rows, gcols, CELLS)
    res.free()
    other.close()
    bm.free()
    sel.free()
    batch.close()


# ---- 3. the limits the cells path lifts ---------------------------------------------------------------------------------------
def test_value_cap_sides(ob, ctx):
    t = cap_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    aggs = [(COUNT, -1), (SUM, 0), (MAX, 0)]
    k1, _, p1 = assert_any(res, [1], aggs, t.cells, range(t.n), "65536", DICT)
    k2, _, p2 = assert_any(res, [2], aggs, t.cells, range(t.n), "65537", CELLS)
    assert len(k1) == CAP and len(k2) == CAP + 1
    with pytest.raises(ob.ObGpuError):
        res.group_by_columns([2], aggs)
    res.free()
    batch.close()


def test_first_capacity_and_refold(ob, ctx):
    """2^20 groups fold once; 2^20 + 1 fold twice (one more launch, and the same groups as the model)"""
    image, (i, key, val) = refold_table()
    batch = ctx.open_batch(image)
    aggs = [(COUNT, -1), (SUM, 2), (MIN, 2), (MAX, 0)]
    launches = []
    for bound in (FIRST_GROUPS, FIRST_GROUPS + 1):
        res = batch.scan(ob.White(0, ob.WHITE_OP_LT, (bound,)), [0])
        before = ctx.launch_count
        keys, got, p = res.group_by_any([1], aggs)
        launches.append(ctx.launch_count - before)
        assert p == CELLS and len(keys) == bound
        uk, want = np_model([key], i < bound, aggs, {0: i, 2: val})
        assert np.array_equal(np.array(keys, dtype=np.int64).reshape(-1), uk.reshape(-1)) and np.array_equal(got, want)
        res.free()
    assert launches[1] == launches[0] + 1, launches
    batch.close()


def test_hashed_tuple_cap(ob, ctx):
    """2^22 tuples: the dictionary fold's hashed path; 2^22 + 1: it refuses, the cells path groups them"""
    image, (i, a, b) = hash_cap_table()
    batch = ctx.open_batch(image)
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0)]
    for flt, sel, path in ((ob.White(0, ob.WHITE_OP_LT, (HASH_GROUPS,)), i < HASH_GROUPS, DICT), (None, i >= 0, CELLS)):
        res = batch.scan(flt, [0])
        keys, got, p = res.group_by_any([1, 2], aggs)
        assert p == path and len(keys) == int(sel.sum())
        uk, want = np_model([a, b], sel, aggs, {0: i})
        assert np.array_equal(np.array(keys, dtype=np.int64), uk) and np.array_equal(got, want)
        res.free()
    batch.close()


# ---- 4. contention and carries ----------------------------------------------------------------------------------------------
def test_contention_and_carries(ob, ctx):
    image, cells = contention_table()
    i = cells[0]
    batch = ctx.open_batch(image)
    aggs = [(COUNT, -1), (SUM, 3), (SUM, 4), (MIN, 3), (MAX, 4), (MIN, 5), (MAX, 5), (COUNT, 5)]
    model_cells = {0: i.tolist(), 1: cells[1].tolist(), 2: cells[2].tolist(), 3: cells[3].tolist(),
                   4: [int(x) for x in cells[4]], 5: cells[5].tolist()}
    for flt, rows in ((None, range(len(i))), (ob.White(0, ob.WHITE_OP_LT, (len(i) // 3,)), range(len(i) // 3))):
        res = batch.scan(flt, [0])
        for gcols in ([1], [2], [2, 1]):
            keys, got, _ = assert_any(res, gcols, aggs, model_cells, rows, (gcols, flt is None), CELLS)
            assert (got[1, :, 1] != 0).all() and (got[2, :, 1] != 0).all()   # every group's sums are past 64 bits
        res.free()
    batch.close()


# ---- 5. the group slot ------------------------------------------------------------------------------------------------------
def test_fetch_groups_of_a_cells_result(ob, ctx):
    t = auto_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    for gc in (1, 2):
        keys, out, p = res.group_by_any([gc], AUTO_AGGS)
        assert p == CELLS
        lib = ob.capi.lib
        n = len(keys)
        hk = np.zeros(n + 1, dtype=np.int64)
        heap = np.zeros(max(sum(len(k[0]) for k in keys if isinstance(k[0], bytes)), 1), dtype=np.uint8)
        ho = np.zeros((len(AUTO_AGGS), max(n, 1), 2), dtype=np.int64)
        assert lib.obgpu_result_fetch_groups(res._h, hk.ctypes.data, heap.ctypes.data, ho.ctypes.data) == 0
        assert np.array_equal(ho[:, :n], out)
        if gc == 1:
            want = [k[0] for k in keys]
            assert [None if k[0] is None else int(v) for k, v in zip(keys, hk[:n])] == want
        else:
            assert [bytes(heap[hk[g]:hk[g + 1]]) for g in range(n)] == [k[0] if k[0] is not None else b"" for k in keys]
    res.free()
    batch.close()


def test_accumulator_merges_both_paths(ob, ctx):
    """a dictionary-only batch (auto_table's first three blocks) and a cells batch (the rest) added to one accumulator equal
    one batch over both"""
    from oceanbase_b200.pipeline import split_table
    t = auto_table()
    parts = split_table(t.image, 3)
    whole = ctx.open_batch(t.image)
    wres = whole.scan(None, [0])
    for gcols in ([1], [1, 2, 3], [2]):
        want_keys, want, _ = wres.group_by_any(gcols, AUTO_AGGS)
        acc = ctx.group_accumulator(len(gcols), AUTO_AGGS)
        paths = []
        for part in parts:
            b = ctx.open_batch(part)
            r = b.scan(None, [0])
            _, _, p = r.group_by_any(gcols, AUTO_AGGS)
            paths.append(p)
            acc.add(r)
            r.free()
            b.close()
        assert paths[0] == DICT and CELLS in paths[1:], paths
        keys, out = acc.fetch()
        acc.free()
        assert keys == want_keys and np.array_equal(out, want), gcols
    wres.free()
    whole.close()


def test_group_and_top_rows_slots_are_independent(ctx):
    t = auto_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    top = res.top_rows([1], [0, 2], 20)
    keys, out, p = res.group_by_any([1, 2], AUTO_AGGS)   # a GROUP BY leaves the rows ...
    assert p == CELLS and res.top_rows([1], [0, 2], 20) == top
    kb = sum(len(k[1]) for k in keys if k[1] is not None)   # ... and the rows leave the groups
    assert res._fetch_group_columns(np.array([1, 2], dtype=np.int32), len(AUTO_AGGS), len(keys), kb)[0] == keys
    res.free()
    batch.close()


# ---- 6. refusals -------------------------------------------------------------------------------------------------------------
def test_refusals(ob, ctx):
    from oceanbase_b200 import capi
    lib = capi.lib
    t = auto_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    cases = [([1], [(SUM_PRODUCT, 0)], capi.OB_NOT_SUPPORTED), ([1], [(SUM, 2)], capi.OB_NOT_SUPPORTED),
             ([1], [(SUM, -1)], capi.OB_INVALID_ARGUMENT), ([9], [(COUNT, -1)], capi.OB_INVALID_ARGUMENT),
             ([-1], [(COUNT, -1)], capi.OB_INVALID_ARGUMENT), ([1, 2, 3, 0, 1], [(COUNT, -1)], capi.OB_INVALID_ARGUMENT),
             ([1], [(COUNT, -1)] * 17, capi.OB_INVALID_ARGUMENT), ([1], [], capi.OB_INVALID_ARGUMENT)]
    for gcols, aggs, code in cases:
        rc, _ = raw_groups(res, "any", gcols, aggs)
        assert rc == code, (gcols, aggs, rc)
        z = np.zeros(64, dtype=np.int64)
        assert lib.obgpu_result_fetch_group_columns(res._h, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data) == capi.OB_INVALID_ARGUMENT
        assert_any(res, [1, 2], AUTO_AGGS, t.cells, range(t.n), "after a refusal", CELLS)
    cols = np.array([1], dtype=np.int32)
    spec = np.array([(COUNT, -1)], dtype=np.int32)
    ng = C.c_int64(0)
    assert lib.obgpu_result_group_by_any(res._h, cols.ctypes.data, 1, spec.ctypes.data, 1, None, C.byref(ng), None) == capi.OB_INVALID_ARGUMENT
    assert lib.obgpu_result_group_by_any(None, cols.ctypes.data, 1, spec.ctypes.data, 1, C.byref(ng), C.byref(ng), None) == capi.OB_INVALID_ARGUMENT
    # a column that is not of one integer or string class in every block: string_table's VARCHAR next to auto_table's INT
    mixed = ob.TableImage.concat([string_table().image, t.image])
    mb = ctx.open_batch(mixed)
    mres = mb.scan(None, [0])
    rc, _ = raw_groups(mres, "any", [1], [(COUNT, -1)])
    assert rc == capi.OB_NOT_SUPPORTED
    assert_any(mres, [0], [(COUNT, -1)], {0: list(range(string_table().n)) + list(range(t.n))},
               range(string_table().n + t.n), "mixed batch, row id key", CELLS)
    mres.free()
    mb.close()
    assert_any(res, [1, 2], AUTO_AGGS, t.cells, range(t.n), "after the mixed batch", CELLS)
    res.free()
    batch.close()
