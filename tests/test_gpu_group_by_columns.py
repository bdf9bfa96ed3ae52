"""GROUP BY over a whole scan keyed by the tuple of values of 1..4 dictionary-coded columns (obgpu_result_group_by_columns /
obgpu_result_fetch_group_columns, ScanResult.group_by_columns) against a plain value model: the selected rows grouped by the
tuple of their true cells, sorted lexicographically over the group columns in the caller's order (each column in its own order,
NULL last within it), each group folded with test_aggregate_exact.fold and encoded as test_gpu_group_by_values.encode encodes a
group. The million-row cases use the same model in numpy. Every comparison is exact.

Cases: 1. every type x codec of the aggregate matrix under five filters, every pair of its group columns, all four PAX group
columns at once, and 2. each group column alone against obgpu_result_group_by_values, byte for byte; 3. every count-kernel path
of path_table with a two-column key; 4. block-varying layouts and formats in one tuple; 5. two string columns (colliding tags,
empty next to NULL, NUL and high bytes, LZ4-stored blocks); 6. NULLs in several columns, a column named twice, no row selected;
7. each fold path at both sides of its limit (test_group_by_columns_shapes proves the sides), the hashed path's cap, the
composite-id overflow and 128-bit carries on the hashed path; 8. rows selected by a column-group bitmap; 9. the bench's cfg3
segment; 10. refusals, bad arguments and the result's group slot."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM, SUM_PRODUCT, M, MATRIX, K, VB, matrix_spec, matrix_table
from test_gpu_aggregate_exact import GROUP_AGGS, PATH_AGGS, PATH_ROWS, path_table
from test_gpu_group_by_values import encode, path_cells, value_model
from test_group_by_columns_shapes import HASH_GROUPS, carry_table, dense_table, hash_cap_table, shared_table, tuple_order
from test_scan_codes_model import (CAP, CS_MODES, TYPE_IDS, auto_table, bench_model, bench_string, bench_workload, cap_table,
                                   concat_table, cs_table, cs_uncodable_table, int_layout_table, open_table, string_table)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def tuple_model(gcells, rows, aggs, cells):
    """(keys, out): the groups of the rows by the tuple (gcells[0][row], ...), in tuple_order"""
    groups = {}
    for r in rows:
        groups.setdefault(tuple(g[r] for g in gcells), []).append(r)
    keys = sorted(groups, key=tuple_order)
    out = np.zeros((len(aggs), len(keys), 2), dtype=np.int64)
    for g, key in enumerate(keys):
        for k, (kind, col) in enumerate(aggs):
            out[k, g] = encode(kind, col, groups[key], cells)
    return keys, out


def assert_tuples(res, gcols, aggs, cells, rows, what):
    got_keys, got = res.group_by_columns(gcols, aggs)
    want_keys, want = tuple_model([cells[c] for c in gcols], list(rows), aggs, cells)
    assert got_keys == want_keys, what
    assert np.array_equal(got, want), what
    return got_keys, got


def assert_same_as_values(res, gc, aggs, what):
    """group_by_columns([gc]) against group_by_values(gc): the same groups, aggregates and fetched bytes"""
    vk, vout = res.group_by_values(gc, aggs)
    ck, cout = res.group_by_columns([gc], aggs)
    assert [k[0] for k in ck] == vk and np.array_equal(cout, vout), what
    assert vout.tobytes() == cout.tobytes(), what


# ---- 1. + 2. every type x codec, every pair of group columns; one column against group_by_values ----------------------------
@pytest.mark.parametrize("tname,codec", MATRIX)
def test_matrix(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    batch = ctx.open_batch(matrix_table(tname, codec))
    n, m, vb = spec.n, spec.truth[M], spec.truth[VB]
    cases = [("no filter", None, range(n)), ("every row", ob.White(K, ob.WHITE_OP_GE, (0,)), range(n)),
             ("M < 40", ob.White(M, ob.WHITE_OP_LT, (40,)), [i for i in range(n) if m[i] < 40]),
             ("no row", ob.White(K, ob.WHITE_OP_LT, (0,)), []),
             ("VB NULL", ob.White(VB, ob.WHITE_OP_NU, ()), [i for i in range(n) if vb[i] is None])]
    gcs = list(spec.group_cols.values())
    keysets = [list(p) for p in itertools.combinations(gcs, 2)] + ([gcs] if len(gcs) == 4 else []) + [gcs[::-1][:2]]
    for what, flt, rows in cases:
        res = batch.scan(flt, [K])
        for gcols in keysets:
            keys, got = assert_tuples(res, gcols, GROUP_AGGS, spec.truth, rows, (gcols, what))
            if what == "no row":
                assert keys == [] and got.shape == (len(GROUP_AGGS), 0, 2)
        for gc in gcs:
            assert_same_as_values(res, gc, GROUP_AGGS, (gc, what))
        res.free()
    batch.close()


# ---- 3. every count-kernel path -----------------------------------------------------------------------------------------------
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
    cases = [("no filter", None, lambda i: True), ("key range", ob.White(0, ob.WHITE_OP_BT, (lo, hi)), lambda i: lo <= i <= hi),
             ("key range and m", ob.And([ob.White(0, ob.WHITE_OP_BT, (lo, hi)), ob.White(1, ob.WHITE_OP_LT, (50,))]),
              lambda i: lo <= i <= hi and m[i] < 50)]
    batch = ctx.open_batch(table)
    for with_index in (False, True):
        batch.set_agg_rows(*agg) if with_index else batch.set_agg_rows(None)
        for what, flt, keep in cases:
            res = batch.scan(flt, [0])
            rows = [i for i in range(n) if keep(i)]
            capped = batch.scan(flt, [0], max_selected_rows=max(len(rows) // 3, 1)) if len(rows) > 1 else None
            for gcols in ([2, 3], [4, 2]):
                keys, got = assert_tuples(res, gcols, PATH_AGGS[1], cells, rows, (what, with_index, gcols))
                if capped is not None:    # the scan overflowed its capacity: its bitmap still selects every row
                    ck, cgot = capped.group_by_columns(gcols, PATH_AGGS[1])
                    assert ck == keys and np.array_equal(cgot, got), (what, with_index, gcols)
            if capped is not None:
                capped.free()
            res.free()
    batch.close()


# ---- 4. block-varying layouts and formats in one tuple ----------------------------------------------------------------------
def check_table(ctx, t, keysets, aggs, image=None, **kw):
    import oceanbase_b200 as ob
    batch = ctx.open_batch(t.image if image is None else image, **kw)
    half = t.n // 2
    for flt, rows in ((None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half])):
        res = batch.scan(flt, [0])
        for gcols in keysets:
            assert_tuples(res, gcols, aggs, t.cells, rows, (t.name, gcols, flt is None))
        res.free()
    batch.close()


@pytest.mark.parametrize("tname", TYPE_IDS)
@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
def test_int_layouts(ctx, tname, byte_packing):
    t = int_layout_table(tname, byte_packing)
    check_table(ctx, t, [[1, 1]], [(COUNT, -1), (COUNT, 1), (SUM, 0), (MIN, 1), (MAX, 1)])


def test_int_layouts_with_strings_and_unsigned(ctx):
    t = open_table()    # 1 INT DICT over every layout, 2 VARCHAR DICT, 3 UINT64 DICT over every layout
    check_table(ctx, t, [[1, 3], [3, 2, 1], [2, 1]], [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (SUM, 3)])


@pytest.mark.parametrize("mode", CS_MODES)
def test_cs_dictionaries(ctx, mode):
    check_table(ctx, cs_table(mode), [[1, 2], [3, 4], [4, 1, 2]], [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (MIN, 2)])


def test_pax_and_cs_in_one_batch(ctx):
    t = concat_table()
    assert t.image.n_blocks > 12
    check_table(ctx, t, [[1, 2], [2, 3, 4], [4, 3, 2, 1]], [(COUNT, -1), (SUM, 1), (MIN, 2), (MAX, 3), (COUNT, 1)])


def test_cs_all_null_block_and_const_refs(ctx):
    check_table(ctx, cs_uncodable_table(), [[1, 2, 3], [3, 1]], [(COUNT, -1), (COUNT, 1), (SUM, 2), (MIN, 3), (MAX, 1)])


# ---- 5. two string columns --------------------------------------------------------------------------------------------------
STR_AGGS = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 4), (COUNT, 4)]


def test_strings(ctx):
    t = string_table()
    check_table(ctx, t, [[1, 2], [2, 1], [2, 4, 1]], STR_AGGS)
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    keys, _ = res.group_by_columns([2, 1], STR_AGGS)
    firsts = [k[0] for k in keys]
    assert b"" in firsts and firsts[-1] is None and firsts.index(b"a\x7fb") < firsts.index(b"a\x80b") < firsts.index(b"a\xffb")
    assert any(k[1] is None for k in keys) and any(k[0] is None for k in keys)
    res.free()
    batch.close()


def test_strings_from_stored_blocks(ob, ctx):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    comp = ob.capi.COMPRESSOR_LZ4
    check_table(ctx, t, [[1, 2], [2, 1]], STR_AGGS, image=compress_table(t.image, comp), compressor=comp)


# ---- 6. NULLs in several columns, a column twice, no row ----------------------------------------------------------------------
def test_nulls_in_several_columns(ob, ctx):
    n = 3000
    rng = np.random.default_rng(23)
    a = [int(x) for x in rng.integers(-3, 4, n)]
    s = [b"k%d" % int(x) for x in rng.integers(0, 5, n)]
    za, zs = rng.random(n) < 0.2, rng.random(n) < 0.2
    w = [int(x) for x in rng.integers(-1000, 1000, n)]
    cols = [ob.Column(5, 0, np.arange(n, dtype=np.int64)), ob.Column(5, 1, np.array(a, dtype=np.int64), nulls=za.astype(np.uint8)),
            ob.Column(22, 1, s, nulls=zs.astype(np.uint8)), ob.Column(5, 0, np.array(w, dtype=np.int64))]
    cells = [list(range(n)), [None if z else v for v, z in zip(a, za)], [None if z else v for v, z in zip(s, zs)], w]
    batch = ctx.open_batch(ob.encode_table(cols, 133))
    aggs = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 3), (COUNT, 1)]
    res = batch.scan(None, [0])
    keys, _ = assert_tuples(res, [1, 2], aggs, cells, range(n), "two columns")
    assert any(k[0] is None and k[1] is not None for k in keys) and any(k[0] is not None and k[1] is None for k in keys)
    assert (None, None) in keys and keys[-1] == (None, None)
    assert_tuples(res, [2, 1], aggs, cells, range(n), "reversed")
    keys, _ = assert_tuples(res, [1, 1], aggs, cells, range(n), "named twice")
    assert all(x == y for x, y in keys)
    keys, _ = assert_tuples(res, [2, 1, 2, 1], aggs, cells, range(n), "four columns, each twice")
    res.free()
    res = batch.scan(ob.White(0, ob.WHITE_OP_LT, (0,)), [0])
    keys, out = res.group_by_columns([1, 2], aggs)
    assert keys == [] and out.shape == (len(aggs), 0, 2)
    res.free()
    batch.close()


# ---- 7. each path at both sides of its limit ------------------------------------------------------------------------------------
def test_shared_and_global_at_the_budget(ctx):
    image, cells = shared_table()
    batch = ctx.open_batch(image)
    n = len(cells[0])
    res = batch.scan(None, [0])
    assert_tuples(res, [1, 2], [(COUNT, -1)], cells, range(n), "shared: 48 KiB exactly")
    assert_tuples(res, [1, 3], [(COUNT, -1)], cells, range(n), "global: just over")
    res.free()
    batch.close()


def test_global_and_hashed_at_dense_limit(ob, ctx):
    image, cells = dense_table()
    batch = ctx.open_batch(image)
    n = len(cells[0])
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0), (MAX, 0)]
    res = batch.scan(ob.White(0, ob.WHITE_OP_LT, (40_000,)), [0])
    assert_tuples(res, [1, 2], aggs, cells, range(40_000), "global: P = 2^20")
    assert_tuples(res, [3, 4], aggs, cells, range(40_000), "hashed: P = 2^20 + 1")
    res.free()
    res = batch.scan(None, [0])
    assert_tuples(res, [3, 4], aggs, cells, range(n), "hashed, every row")
    res.free()
    batch.close()


def np_model(keys, sel, aggs, vals):
    """the tuple model in numpy for columns without NULLs: keys int64 arrays (in their columns' order), vals the aggregate
    columns (int64, or uint64 for unsigned); returns (unique keys [G][n_cols], out [n_aggs][G][2])"""
    ks = np.stack([k[sel] for k in keys], axis=1)
    uk, inv = np.unique(ks, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(inv, kind="stable")
    starts = np.searchsorted(inv[order], np.arange(len(uk)))
    counts = np.bincount(inv, minlength=len(uk)).astype(np.int64)
    out = np.zeros((len(aggs), len(uk), 2), dtype=np.int64)
    for k, (kind, col) in enumerate(aggs):
        if kind == COUNT:
            out[k, :, 0] = counts
            continue
        v = vals[col][sel][order]
        if kind in (MIN, MAX):
            f = np.minimum if kind == MIN else np.maximum
            out[k, :, 0] = f.reduceat(v, starts).view(np.int64)
            out[k, :, 1] = 1
            continue
        u = v.view(np.uint64)
        lo = np.add.reduceat((u & np.uint64(0xffffffff)).astype(np.int64), starts)
        hi = np.add.reduceat((v >> 32).astype(np.int64) if v.dtype == np.int64 else (u >> np.uint64(32)).astype(np.int64), starts)
        hl = (hi.view(np.uint64) & np.uint64(0xffffffff)) << np.uint64(32)
        x = hl + lo.view(np.uint64)
        out[k, :, 0] = x.view(np.int64)
        out[k, :, 1] = (hi >> 32) + (x < hl).astype(np.int64)
    return uk, out


def test_hashed_cap(ob, ctx):
    image, (i, a, b) = hash_cap_table()
    batch = ctx.open_batch(image)
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0)]
    res = batch.scan(ob.White(0, ob.WHITE_OP_LT, (HASH_GROUPS,)), [0])
    keys, got = res.group_by_columns([1, 2], aggs)
    assert len(keys) == HASH_GROUPS
    sel = i < HASH_GROUPS
    uk, want = np_model([a, b], sel, aggs, {0: i})
    assert np.array_equal(np.array(keys, dtype=np.int64), uk) and np.array_equal(got, want)
    res.free()
    res = batch.scan(None, [0])
    with pytest.raises(ob.ObGpuError) as e:
        res.group_by_columns([1, 2], aggs)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    keys, got = res.group_by_columns([2], [(COUNT, -1)])     # the ctx and the result still work
    assert keys == [(v,) for v in range(2049)] and got[0, :, 0].tolist() == [2048] * 2048 + [1]
    res.free()
    batch.close()


def test_composite_id_overflow(ob, ctx):
    t = cap_table()
    batch = ctx.open_batch(t.image)
    res = batch.scan(None, [0])
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0), (MAX, 0)]
    with pytest.raises(ob.ObGpuError) as e:
        res.group_by_columns([1, 1, 1, 1], aggs)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    keys, _ = assert_tuples(res, [1, 1, 1], aggs, t.cells, range(t.n), "three times: hashed, ids above 2^48")
    assert len(keys) == CAP
    res.free()
    batch.close()


def test_carries_on_the_hashed_path(ob, ctx):
    image, (m, g1, g2, g3, a, u) = carry_table()
    aggs = [(COUNT, -1), (SUM, 4), (SUM, 5), (MIN, 5), (MAX, 5), (MIN, 4), (MAX, 4)]
    batch = ctx.open_batch(image)
    for flt, sel in ((None, np.ones(len(m), dtype=bool)), (ob.White(0, ob.WHITE_OP_LT, (50,)), m < 50)):
        res = batch.scan(flt, [0])
        keys, got = res.group_by_columns([1, 2, 3], aggs)
        uk, want = np_model([g1, g2, g3], sel, aggs, {4: a, 5: u})
        assert np.array_equal(np.array(keys, dtype=np.int64), uk)
        assert np.array_equal(got, want), flt is None
        assert (got[1, :, 1] > 0).sum() >= 30 and (got[2, :, 1] > 0).sum() >= 30     # 128-bit sums that carried
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
    for gcols in ([2, 3], [3, 4, 2]):
        assert_tuples(res, gcols, PATH_AGGS[1], cells, rows, ("bitmap", gcols))
    res.free()
    batch.close()
    sel.free()
    other.close()
    bm.free()


# ---- 9. the bench's cfg3 segment --------------------------------------------------------------------------------------------
def test_bench_segment(ctx):
    w = bench_workload()
    ints, strs = bench_model()
    n = w.table.total_rows
    cells = {c: ints[c][0][ints[c][1][:n]].tolist() for c in (0, 1, 3)}
    cells[8] = [bench_string(strs, 8, int(k)) for k in strs[8][1][:n].tolist()]
    batch = ctx.open_batch(w.table)
    res = batch.scan(None, [0])
    aggs = [(COUNT, -1), (SUM, 1), (MIN, 1), (MAX, 1)]
    for gcols in ([0, 8], [0, 3]):
        keys, _ = assert_tuples(res, gcols, aggs, cells, range(n), ("cfg3", gcols))
        assert len(keys) == len(set(zip(*[cells[c] for c in gcols])))
    res.free()
    batch.close()


# ---- 10. refusals, arguments and the result's group slot --------------------------------------------------------------------
def test_refusals_and_arguments(ob, ctx):
    lib = ob.capi.lib
    a = auto_table()
    batch = ctx.open_batch(a.image)
    res = batch.scan(None, [0])
    ng, kb, hn = C.c_int64(), C.c_int64(), C.c_int32()
    keys, nulls, out = np.zeros(64, dtype=np.int64), np.zeros(64, dtype=np.uint8), np.zeros(256, dtype=np.int64)
    heap = np.zeros(64, dtype=np.uint8)

    def call(gcols, aggs, cols_ptr=True, outs=True):
        g = np.array(gcols, dtype=np.int32)
        spec = np.array(aggs, dtype=np.int32).reshape(-1, 2)
        return lib.obgpu_result_group_by_columns(res._h, g.ctypes.data if cols_ptr else None, len(gcols), spec.ctypes.data if len(aggs) else None,
                                                 len(aggs), C.byref(ng) if outs else None, C.byref(kb))

    def fetch_columns():
        return lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data)

    def fetch_groups():
        return lib.obgpu_result_fetch_groups(res._h, keys.ctypes.data, heap.ctypes.data, out.ctypes.data)

    assert fetch_columns() == ob.OB_INVALID_ARGUMENT       # before any group-by on this result
    ok = [(COUNT, -1)]
    for gcols in ([1, 3], [3, 1], [3, 2], [3, 3, 1]):      # OBGPU_ENC_AUTO columns with RAW blocks, in any position
        assert call(gcols, ok) == ob.OB_NOT_SUPPORTED, gcols
        assert fetch_columns() == ob.OB_INVALID_ARGUMENT and fetch_groups() == ob.OB_INVALID_ARGUMENT
    assert call([3, 3], [(SUM_PRODUCT, 0)]) == ob.OB_NOT_SUPPORTED
    assert call([3, 3], [(SUM, 2)]) == ob.OB_NOT_SUPPORTED          # a string aggregate column
    assert call([3, 3], []) == ob.OB_INVALID_ARGUMENT
    assert call([3, 3], ok * 17) == ob.OB_INVALID_ARGUMENT
    assert call([], ok) == ob.OB_INVALID_ARGUMENT
    assert call([3] * 5, ok) == ob.OB_INVALID_ARGUMENT
    assert call([3, 4], ok) == ob.OB_INVALID_ARGUMENT and call([-1, 3], ok) == ob.OB_INVALID_ARGUMENT
    assert call([3, 3], ok, cols_ptr=False) == ob.OB_INVALID_ARGUMENT
    assert call([3, 3], ok, outs=False) == ob.OB_INVALID_ARGUMENT
    assert fetch_columns() == ob.OB_INVALID_ARGUMENT
    assert_tuples(res, [3, 3], ok * 16, a.cells, range(a.n), "16 aggregates after the refusals")
    # the slot: fetch_groups refuses two-column groups; fetch_group_columns takes group_by_values' own
    assert call([3, 3], ok) == 0
    assert fetch_groups() == ob.OB_INVALID_ARGUMENT
    spec = np.array(ok, dtype=np.int32)
    assert lib.obgpu_result_group_by_values(res._h, 3, spec.ctypes.data, 1, C.byref(ng), C.byref(kb), C.byref(hn)) == 0
    assert fetch_columns() == 0
    vk, vout = value_model(a.cells[3], range(a.n), ok, a.cells)
    g = ng.value
    assert keys[:g].tolist() == vk and not nulls[:g].any() and np.array_equal(out[:2 * g].reshape(1, g, 2), vout)
    assert fetch_groups() == 0
    res.free()
    batch.close()
