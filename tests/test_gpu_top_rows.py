"""ORDER BY ... LIMIT k over a whole scan (obgpu_result_top_rows / obgpu_result_fetch_top_rows, ScanResult.top_rows) against a
plain Python model: the selected rows sorted by (key tuple with DESC and NULL placement, block, row) over the generator's cells,
sliced to k. Positions, output values, NULLs and string bytes must match exactly.

Cases: 1. every integer type (1-, 4- and 8-byte datums, signed and unsigned, DATE and YEAR, with their extremes) under every
integer codec of the aggregate matrix (PAX RAW byte- and bit-packed, DICT, RLE, CONST, INTEGER_BASE_DIFF, CS INTEGER and
INT_DICT), ASC / DESC x NULLS FIRST / LAST, 1..4 keys and a column named twice, k from 1 past the selection, three filters;
2. every string codec of the string matrix (PAX var and fixed, DICT, RLE, CONST, HEX, STRING_DIFF, STRING_PREFIX, the span
columns, CS STRING and STR_DICT) with shared 8-byte prefixes, proper prefixes, the empty string and NUL bytes; 3. block-varying
layouts: OBGPU_ENC_AUTO, CS dictionaries under three stream codecs, a PAX + CS batch, every INT layout; 4. LZ4-, zstd- and
zlib-stored blocks; 5. k at 65 536 and the 65 537 refusal, an all-equal key where position alone decides, a 16-value key with
k >> 16; 6. a capacity-overflowed scan, a column-group bitmap and an empty selection; 7. the bench's cfg3 segment; 8. refusals,
each leaving the slot empty and the ctx usable, and the top-rows slot independent of the group slot."""
import ctypes as C
import functools

import numpy as np
import pytest

from test_aggregate_exact import COUNT, K, M, MATRIX, VA, VB, VN, W, matrix_spec, matrix_table
from test_scan_codes_model import (CS_MODES, TYPE_IDS, auto_table, bench_model, bench_string, bench_workload, concat_table, cs_table,
                                   int_layout_table, string_table)
import test_string_filter_exact as sfe
from test_top_rows_shapes import big_table

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


def positions(batch):
    """(block, row) of every row of the batch, in the batch's row order"""
    out = []
    for b in range(batch.n_blocks):
        out += [(b, r) for r in range(batch.block_info(b)[0])]
    return out


def norm(keys):
    return [(k, 0, 0) if isinstance(k, int) else k for k in keys]


def model_order(cells, rows, keys, pos):
    """the rows in ORDER BY keys order, ties by position"""
    keys = norm(keys)

    def cmp(i, j):
        for col, desc, nf in keys:
            a, b = cells[col][i], cells[col][j]
            if a is None or b is None:
                if a is None and b is None:
                    continue
                return (-1 if a is None else 1) if nf else (1 if a is None else -1)
            if a != b:
                c = -1 if a < b else 1
                return -c if desc else c
        return -1 if pos[i] < pos[j] else (1 if pos[i] > pos[j] else 0)
    return sorted(rows, key=functools.cmp_to_key(cmp))


def check(res, cells, order, keys, out_cols, k, pos, what):
    got_pos, got_rows = res.top_rows(keys, out_cols, k)
    want = order[:k]
    assert got_pos == [pos[i] for i in want], what
    assert got_rows == [tuple(cells[c][i] for c in out_cols) for i in want], what


def check_many(res, cells, rows, keysets, out_cols, ks, pos, what):
    rows = list(rows)
    n = len(rows)
    for keys in keysets:
        order = model_order(cells, rows, keys, pos)
        for k in sorted({kk for kk in ks(n) if kk >= 1}):
            check(res, cells, order, keys, out_cols, k, pos, (what, keys, k))


def small_ks(n):
    return (1, 2, 7, n - 1, n, n + 5)


# ---- 1. every integer type x codec ---------------------------------------------------------------------------------------------
INT_KEYSETS = [[VA], [(VA, 1, 1)], [(VB, 0, 1)], [(VB, 1, 0)], [(W, 1, 0), (VA, 0, 0)], [(M, 0, 0), (VB, 1, 1), (VB, 0, 0)],
               [(VN, 0, 1), (M, 1, 0), (W, 0, 1), (VA, 1, 0)]]


@pytest.mark.parametrize("tname,codec", MATRIX)
def test_int_matrix(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    batch = ctx.open_batch(matrix_table(tname, codec))
    pos = positions(batch)
    n, m = spec.n, spec.truth[M]
    cases = [("no filter", None, range(n)), ("M < 40", ob.White(M, ob.WHITE_OP_LT, (40,)), [i for i in range(n) if m[i] < 40]),
             ("no row", ob.White(K, ob.WHITE_OP_LT, (0,)), [])]
    for what, flt, rows in cases:
        res = batch.scan(flt, [K])
        check_many(res, spec.truth, rows, INT_KEYSETS, [K, VA, VB, VN, W], small_ks, pos, (tname, codec, what))
        res.free()
    batch.close()


# ---- 2. every string codec -----------------------------------------------------------------------------------------------------
STR_KEYSETS = [[sfe.S], [(sfe.S, 1, 1)], [(sfe.S, 0, 1), (sfe.TCOL, 1, 0)], [(sfe.TCOL, 0, 0), (sfe.S, 1, 0), sfe.K]]


@pytest.mark.parametrize("codec,tname,nname", sfe.MATRIX, ids=sfe.MATRIX_IDS)
def test_string_matrix(ob, ctx, codec, tname, nname):
    spec = sfe.spec_of(codec, tname, nname)
    batch = ctx.open_batch(sfe.table_of(codec, tname, nname))
    pos = positions(batch)
    n, m = spec.n, spec.truth[sfe.M]
    for flt, rows in ((None, range(n)), (ob.White(sfe.M, ob.WHITE_OP_LT, (30,)), [i for i in range(n) if m[i] < 30])):
        res = batch.scan(flt, [sfe.K])
        check_many(res, spec.truth, rows, STR_KEYSETS, [sfe.S, sfe.K, sfe.TCOL], lambda n: (1, 50, n), pos, (codec, tname, nname))
        res.free()
    batch.close()


# ---- 3. + 4. block-varying layouts and stored blocks -------------------------------------------------------------------------
def check_table(ctx, t, keysets, out_cols, image=None, **kw):
    import oceanbase_b200 as ob
    batch = ctx.open_batch(t.image if image is None else image, **kw)
    pos = positions(batch)
    half = t.n // 2
    for flt, rows in ((None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half])):
        res = batch.scan(flt, [0])
        check_many(res, t.cells, rows, keysets, out_cols, lambda n: (1, 33, n - 1, n + 1), pos, (t.name, flt is None))
        res.free()
    batch.close()


def test_auto_table(ctx):
    check_table(ctx, auto_table(), [[1], [(2, 1, 0)], [(3, 0, 0), (2, 1, 1)], [(3, 1, 0), (1, 0, 0), (2, 0, 0), (3, 0, 0)]], [1, 2, 3])


@pytest.mark.parametrize("mode", CS_MODES)
def test_cs_tables(ctx, mode):
    check_table(ctx, cs_table(mode), [[3], [(3, 1, 1)], [(4, 0, 1), (1, 1, 0)], [(2, 0, 0), (4, 1, 0), (3, 0, 1)]], [1, 2, 3, 4])


def test_pax_and_cs_in_one_batch(ctx):
    check_table(ctx, concat_table(), [[(3, 1, 0)], [(4, 0, 1), (2, 0, 0)]], [4, 3, 2, 1])


@pytest.mark.parametrize("tname", TYPE_IDS)
@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
def test_int_layouts(ctx, tname, byte_packing):
    check_table(ctx, int_layout_table(tname, byte_packing), [[1], [(1, 1, 1)], [(1, 0, 1), (0, 1, 0)]], [1, 0])


def test_strings(ctx):
    check_table(ctx, string_table(), [[1], [(2, 1, 1)], [(2, 0, 0), (1, 1, 0)], [(4, 0, 0), (2, 0, 1), (1, 0, 0)]], [1, 2, 4])


@pytest.mark.parametrize("comp", ["lz4", "zstd", "zlib"])
def test_stored_blocks(ob, ctx, comp):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    c = {"lz4": ob.capi.COMPRESSOR_LZ4, "zstd": ob.capi.COMPRESSOR_ZSTD_1_3_8, "zlib": ob.capi.COMPRESSOR_ZLIB}[comp]
    check_table(ctx, t, [[(1, 1, 0)], [(2, 0, 1), (1, 0, 0)]], [1, 2, 3], image=compress_table(t.image, c), compressor=c)


# ---- 5. k at its limit, all-equal and 16-value keys --------------------------------------------------------------------------
def test_k_limits_and_ties(ob, ctx):
    image, cells = big_table()
    n = len(cells[0])
    batch = ctx.open_batch(image)
    pos = positions(batch)
    res = batch.scan(None, [0])
    got_pos, got_rows = res.top_rows([1], [0], 65536)                  # all equal: position alone decides
    assert got_pos == pos[:65536] and got_rows == [(i,) for i in range(65536)]
    got_pos, _ = res.top_rows([(1, 1, 0)], [], 65536)
    assert got_pos == pos[:65536]
    v2 = np.array(cells[2])
    for desc in (0, 1):
        order = np.lexsort((np.arange(n), -v2 if desc else v2))     # 16 values, k >> 16: ties across the threshold
        for k in (1000, 65536):
            got_pos, got_rows = res.top_rows([(2, desc, 0)], [2, 0], k)
            assert got_pos == [pos[i] for i in order[:k]] and got_rows == [(cells[2][i], i) for i in order[:k]], (desc, k)
    order = sorted(range(n), key=lambda i: (cells[3][i], -cells[2][i], i))
    got_pos, got_rows = res.top_rows([3, (2, 1, 0)], [3], 1000)       # a string first key whose ties pass 8 bytes
    assert got_pos == [pos[i] for i in order[:1000]] and got_rows == [(cells[3][i],) for i in order[:1000]]
    with pytest.raises(ob.ObGpuError):
        res.top_rows([1], [0], 65537)
    assert ctx.last_error()
    got_pos, _ = res.top_rows([1], [0], 3)                              # the ctx is still usable
    assert got_pos == pos[:3]
    res.free()
    batch.close()


# ---- 6. overflowed scan, bitmap scan, empty selection --------------------------------------------------------------------------
def test_overflow_bitmap_and_empty(ob, ctx):
    spec = matrix_spec("int", "dict")
    table = matrix_table("int", "dict")
    batch = ctx.open_batch(table)
    pos = positions(batch)
    n, m = spec.n, spec.truth[M]
    flt = ob.White(M, ob.WHITE_OP_LT, (30,))
    rows = [i for i in range(n) if m[i] < 30]
    capped = batch.scan(flt, [K], max_selected_rows=len(rows) // 3)
    check_many(capped, spec.truth, rows, INT_KEYSETS[:3], [K, VA], lambda n: (1, 9, n), pos, "capped")
    capped.free()
    bm = ob.CGBitmap(ctx, n)
    sel = batch.scan(flt, [K])
    bm.apply(sel, 0, "set")
    other = ctx.open_batch(table)
    res = other.scan_bitmap(bm, [K])
    check_many(res, spec.truth, rows, INT_KEYSETS[:3], [K, VB], lambda n: (1, 9, n), pos, "bitmap")
    res.free()
    other.close()
    bm.free()
    sel.free()
    none = batch.scan(ob.White(K, ob.WHITE_OP_LT, (0,)), [K])
    assert none.top_rows([VA], [VA, K], 5) == ([], [])
    assert none.top_rows([VA], [], 1) == ([], [])
    none.free()
    batch.close()


# ---- 7. the bench's cfg3 segment ---------------------------------------------------------------------------------------------
def test_bench_segment(ctx):
    w = bench_workload()
    ints, strs = bench_model()
    n = w.table.total_rows
    cells = {c: ints[c][0][ints[c][1][:n]].tolist() for c in (0, 1, 3)}
    cells[8] = [bench_string(strs, 8, int(k)) for k in strs[8][1][:n].tolist()]
    batch = ctx.open_batch(w.table)
    pos = positions(batch)
    res = batch.scan(None, [0])
    idx = np.arange(n)
    c3, c0 = np.array(cells[3]), np.array(cells[0])
    for keys, order, k in (([(3, 1, 0)], np.lexsort((idx, -c3)), 10_000), ([0], np.lexsort((idx, c0)), 1000)):
        got_pos, got_rows = res.top_rows(keys, [1, 8], k)
        assert got_pos == [pos[i] for i in order[:k]], keys
        assert got_rows == [(cells[1][i], cells[8][i]) for i in order[:k]], keys
    order = sorted(range(n), key=lambda i: (cells[8][i], cells[1][i], i))[:100]
    got_pos, got_rows = res.top_rows([8, 1], [1, 8], 100)
    assert got_pos == [pos[i] for i in order] and got_rows == [(cells[1][i], cells[8][i]) for i in order]
    res.free()
    batch.close()


# ---- 8. refusals and the slots -----------------------------------------------------------------------------------------------
def test_refusals_and_slots(ob, ctx):
    lib = ob.capi.lib
    t = string_table()
    batch = ctx.open_batch(t.image)
    pos = positions(batch)
    res = batch.scan(None, [0])
    nr, hb = C.c_int64(), C.c_int64()
    blk, row = np.zeros(64, dtype=np.int32), np.zeros(64, dtype=np.int32)
    vals, nulls, heap = np.zeros(1024, dtype=np.int64), np.zeros(1024, dtype=np.uint8), np.zeros(1 << 16, dtype=np.uint8)

    def call(keys, outs, k, keys_ptr=True, outs_ptr=True, n_ptr=True):
        ka = np.array(norm(keys), dtype=np.int32).reshape(-1, 3)
        oa = np.array(outs, dtype=np.int32)
        return lib.obgpu_result_top_rows(res._h, ka.ctypes.data if keys_ptr else None, len(keys), oa.ctypes.data if outs_ptr else None,
                                         len(outs), k, C.byref(nr) if n_ptr else None, C.byref(hb))

    def fetch():
        return lib.obgpu_result_fetch_top_rows(res._h, blk.ctypes.data, row.ctypes.data, vals.ctypes.data, nulls.ctypes.data, heap.ctypes.data)

    assert fetch() == ob.OB_INVALID_ARGUMENT                     # before any call
    order = model_order(t.cells, range(t.n), [2], pos)
    bad = [(([], [1], 5), ob.OB_INVALID_ARGUMENT), (([1] * 5, [1], 5), ob.OB_INVALID_ARGUMENT),
           (([1], [1] * 17, 5), ob.OB_INVALID_ARGUMENT), (([1], [1], 0), ob.OB_INVALID_ARGUMENT), (([1], [1], -3), ob.OB_INVALID_ARGUMENT),
           (([5], [1], 5), ob.OB_INVALID_ARGUMENT), (([-1], [1], 5), ob.OB_INVALID_ARGUMENT), (([1], [5], 5), ob.OB_INVALID_ARGUMENT),
           (([1], [1], 65537), ob.OB_NOT_SUPPORTED)]
    for args, code in bad:
        assert call([2], [1], 4) == 0 and fetch() == 0          # a good call fills the slot ...
        assert call(*args) == code, args                          # ... and a refused one empties it
        assert fetch() == ob.OB_INVALID_ARGUMENT, args
        check(res, t.cells, order, [2], [1, 2], 6, pos, args)    # the ctx is usable
    for kw in ({"keys_ptr": False}, {"outs_ptr": False}, {"n_ptr": False}):
        assert call([2], [1], 4, **kw) == ob.OB_INVALID_ARGUMENT, kw
        assert fetch() == ob.OB_INVALID_ARGUMENT
    assert call([2], [], 4, outs_ptr=False) == 0 and fetch() == 0     # no output column: no pointer needed
    # a column that is not an integer or string class in every block: the auto table's INT column is fine, a mixed batch is not
    mixed = ob.TableImage.concat([t.image, auto_table().image])
    mb = ctx.open_batch(mixed)
    mres = mb.scan(None, [0])
    for keys, outs in (([1], [0]), ([0], [1]), ([(0, 1, 0), (1, 0, 0)], [])):
        with pytest.raises(ob.ObGpuError) as e:
            mres.top_rows(keys, outs, 3)
        assert e.value.code == ob.OB_NOT_SUPPORTED, (keys, outs)
    got_pos, got_rows = mres.top_rows([0], [0], 3)               # both parts number their rows from 0: row 0 ties across them
    assert got_pos == [(0, 0), (t.image.n_blocks, 0), (0, 1)] and got_rows == [(0,), (0,), (1,)]
    mres.free()
    mb.close()
    # the slots: a GROUP BY leaves the rows, the rows leave the groups
    gk, gout = res.group_by_values(4, [(COUNT, -1)])
    check(res, t.cells, model_order(t.cells, range(t.n), [(1, 1, 1)], pos), [(1, 1, 1)], [1, 4], 20, pos, "after group by")
    keys = np.zeros(64, dtype=np.int64)
    out = np.zeros(256, dtype=np.int64)
    gheap = np.zeros(64, dtype=np.uint8)
    assert call([(1, 1, 1)], [1, 4], 20) == 0
    assert lib.obgpu_result_fetch_groups(res._h, keys.ctypes.data, gheap.ctypes.data, out.ctypes.data) == 0
    assert keys[:len(gk)].tolist() == gk and out[:2 * len(gk)].reshape(1, -1, 2).tolist() == gout.tolist()
    assert res.group_by_values(4, [(COUNT, -1)])[0] == gk
    assert fetch() == 0 and nr.value == 20
    res.free()
    batch.close()


# ---- TIME, beside DATE and YEAR of the matrix --------------------------------------------------------------------------------
def test_time_type(ob, ctx):
    n = 1200
    rng = np.random.default_rng(41)
    ext = [-(1 << 63), (1 << 63) - 1, -1, 0, 1, -838 * 3600 * 10 ** 6, 838 * 3600 * 10 ** 6]
    vals = [ext[i % len(ext)] if i % 9 == 0 else int(x) for i, x in enumerate(rng.integers(-(1 << 40), 1 << 40, n))]
    z = (rng.random(n) < 0.1).astype(np.uint8)
    cells = [list(range(n)), [None if zz else v for v, zz in zip(vals, z.tolist())]]
    for enc in (ob.ENC_RAW, ob.ENC_DICT):
        cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, np.arange(n, dtype=np.int64)),
                ob.Column(ob.capi.OBJ_TIME, enc, np.array(vals if enc == ob.ENC_RAW else [v % 97 - 48 for v in vals], dtype=np.int64),
                          nulls=z)]
        if enc == ob.ENC_DICT:
            cells[1] = [None if zz else v % 97 - 48 for v, zz in zip(vals, z.tolist())]
        batch = ctx.open_batch(ob.encode_table(cols, 250))
        pos = positions(batch)
        res = batch.scan(None, [0])
        check_many(res, cells, range(n), [[1], [(1, 1, 1)], [(1, 0, 1), (0, 1, 0)]], [1, 0], lambda n: (1, 40, n), pos, ("time", enc))
        res.free()
        batch.close()
