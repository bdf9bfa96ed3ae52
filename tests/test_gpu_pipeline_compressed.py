"""Stored (compressed) micro-blocks through the host pipeline, and string cells returned as bytes in caller heaps.

The stored-form pipeline (obgpu_host_scan_spec.compressor_type) must give what the plain-image pipeline and the oracle give:
integers byte for byte, NULL words, batch slices, the four aggregate kinds, and string cells as bytes, over PAX tables of every
codec (the rebuilt HEX_PACKING / STRING_DIFF / STRING_PREFIX columns included) and CS tables, with incompressible blocks
stored raw next to compressed ones. obgpu_result_string_bytes / obgpu_result_fetch_string_heap are checked directly too:
several columns, NULL and empty cells, windows, argument checks and a launch count that does not depend on rows or columns."""
import ctypes as C

import numpy as np
import pytest

import oracle_binding as ora
from test_string_codecs import pick

pytestmark = pytest.mark.gpu

COMPRESSORS = [1, 2, 4, 6, 7]   # NONE, LZ4, ZLIB, ZSTD_1_3_8, LZ4_1_9_1


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


def _tables(ob):
    """{name: (table, column values, string columns)}; the first two blocks of each table are high-entropy (stored raw)."""
    n, rpb = 16_000, 400
    rng = np.random.default_rng(21)
    nl = (rng.random(n) < 0.1).astype(np.uint8)
    noise_rows = 2 * rpb
    key = np.arange(n, dtype=np.int64) * 3 + 1
    small = rng.integers(0, 50, size=n, dtype=np.int64)
    runs = np.repeat(np.arange(n // 100 + 1, dtype=np.int64), 100)[:n]
    wide = rng.integers(-(1 << 62), 1 << 62, size=n, dtype=np.int64)
    wide[noise_rows:] %= 1000
    noise = [bytes(rng.integers(0, 256, size=160, dtype=np.uint8)) if i < noise_rows else (b"" if i % 3 else b"q%d" % (i % 9))
             for i in range(n)]
    words = [b"w%03d" % (i % 37) for i in range(n)]
    hexs = [pick(rng, b"0123456789abcdef", int(rng.integers(0, 20))) for _ in range(n)]
    diffs = [b"ORDER-2024-" + pick(rng, b"0123456789", 5) + b"-X" for _ in range(n)]
    pre = [[b"http://www.example.com/", b"https://oceanbase.com/docs/", b""][int(rng.integers(0, 3))] +
           bytes(rng.integers(97, 123, size=int(rng.integers(0, 12)), dtype=np.uint8)) for _ in range(n)]
    C_ = ob.Column
    pax = [C_(ob.OBJ_INT, ob.ENC_RAW, key), C_(ob.OBJ_INT, ob.ENC_RAW, small, nulls=nl), C_(ob.OBJ_INT, ob.ENC_DICT, small),
           C_(ob.OBJ_INT, ob.ENC_RLE, runs), C_(ob.OBJ_INT, ob.ENC_CONST, np.full(n, 7, dtype=np.int64)),
           C_(ob.OBJ_INT, ob.ENC_INTEGER_BASE_DIFF, wide), C_(ob.OBJ_VARCHAR, ob.ENC_RAW, noise, nulls=nl),
           C_(ob.OBJ_VARCHAR, ob.ENC_DICT, words), C_(ob.OBJ_VARCHAR, ob.ENC_HEX_PACKING, hexs, nulls=nl),
           C_(ob.OBJ_VARCHAR, ob.ENC_STRING_DIFF, diffs), C_(ob.OBJ_VARCHAR, ob.ENC_STRING_PREFIX, pre, nulls=nl)]
    cs = [C_(ob.OBJ_INT, ob.ENC_CS_INTEGER, key), C_(ob.OBJ_INT, ob.ENC_CS_INTEGER, small, nulls=nl),
          C_(ob.OBJ_INT, ob.ENC_CS_INT_DICT, small), C_(ob.OBJ_INT, ob.ENC_CS_INTEGER, wide),
          C_(ob.OBJ_VARCHAR, ob.ENC_CS_STRING, noise, nulls=nl), C_(ob.OBJ_VARCHAR, ob.ENC_CS_STR_DICT, words, nulls=nl)]
    vals = {"pax": [key, small, small, runs, None, wide, noise, words, hexs, diffs, pre], "cs": [key, small, small, wide, noise, words]}
    nulls = {"pax": [None, nl, None, None, None, None, nl, None, nl, None, nl], "cs": [None, nl, None, None, nl, nl]}
    return {"pax": (ob.encode_table(pax, rpb, rowkey_cnt=1), vals["pax"], nulls["pax"], [6, 7, 8, 9, 10]),
            "cs": (ob.encode_table(cs, rpb, rowkey_cnt=1), vals["cs"], nulls["cs"], [4, 5])}


@pytest.fixture(scope="module")
def tables(ob):
    return _tables(ob)


@pytest.fixture(scope="module")
def pipe():
    from oceanbase_b200.pipeline import HostScanPipeline
    p = HostScanPipeline(0, n_workers=3)
    yield p
    p.close()


def _filter(ob, name):
    # an integer leaf and a string leaf
    return ob.And([ob.White(1, ob.WHITE_OP_LT, (35,)), ob.White(7 if name == "pax" else 5, ob.WHITE_OP_NE, (b"w003",))])


def _ints(out, c):
    return np.concatenate([b.cols[c] for b in out.batches]) if out.batches else np.zeros(0)


def _nulls(out, c):
    bits = []
    for b in out.batches:
        w = b.nulls[c]
        bits.append(np.array([(int(w[k >> 6]) >> (k & 63)) & 1 for k in range(b.selected_rows)], dtype=np.uint8))
    return np.concatenate(bits) if bits else np.zeros(0, dtype=np.uint8)


def _strings(out, c):
    return [s for b in out.batches for s in b.strings(c)]


def _same(a, b, proj_str):
    assert a.selected_rows == b.selected_rows and a.total_rows == b.total_rows
    assert [(x.block_begin, x.block_end, x.selected_rows) for x in a.batches] == [(x.block_begin, x.block_end, x.selected_rows) for x in b.batches]
    for c, s in enumerate(proj_str):
        assert np.array_equal(_nulls(a, c), _nulls(b, c)), c
        if s:
            assert _strings(a, c) == _strings(b, c), c
        else:
            assert np.array_equal(_ints(a, c), _ints(b, c)), c
    assert a.aggregates == b.aggregates


@pytest.mark.parametrize("name", ["pax", "cs"])
@pytest.mark.parametrize("comp", COMPRESSORS)
def test_stored_pipeline_equals_plain_and_oracle(ob, tables, name, comp):
    from oceanbase_b200.pipeline import HostScanPipeline
    from oceanbase_b200.sstable import compress_table
    import lz4_ref
    table, vals, nulls, str_cols = tables[name]
    stored = compress_table(table, comp)
    fields = [lz4_ref.header_fields(stored.block(i)) for i in range(stored.n_blocks)]
    raw = sum(1 for f in fields if f[2] == f[1])
    if comp != 1:
        assert raw < stored.n_blocks
    proj = list(range(len(vals)))
    proj_str = [c in str_cols for c in proj]
    aggs = [(ob.AGG_COUNT, 1, -1), (ob.AGG_SUM, 5 if name == "pax" else 3, -1), (ob.AGG_SUM_PRODUCT, 0, 1), (ob.AGG_MIN, 1, -1),
            (ob.AGG_MAX, 0, -1)]
    workers, ramp, hint = [(1, 0, 1.0), (3, 2, 0.02), (3, 0, 0.3), (1, 2, 0.01), (3, 2, 1.0)][COMPRESSORS.index(comp)]
    p = HostScanPipeline(0, n_workers=workers)
    try:
        for flt in (_filter(ob, name), None):
            plain = p.scan(table, flt, proj, blocks_per_batch=7, selectivity_hint=hint, ramp=ramp, aggs=aggs, heap_bytes=0)
            got = p.scan(stored, flt, proj, blocks_per_batch=7, selectivity_hint=hint, ramp=ramp, aggs=aggs, compressor=comp)
            _same(plain, got, proj_str)
            assert got.h2d_bytes == stored.image.size   # the stored bytes, copied once
            assert got.d2h_bytes > 0
            if flt is None:   # every row in order: the generated cells
                for c in str_cols:
                    want = [None if (nulls[c] is not None and nulls[c][i]) else bytes(vals[c][i]) for i in range(table.total_rows)]
                    assert _strings(got, c) == want, c
            # the oracle over the plain image: integer columns and string bytes (ordinary string columns)
            want = ora.scan_table(table, flt, proj, proj_str, [8] * len(proj))
            assert got.selected_rows == want["selected"]
            for c in proj:
                if not proj_str[c]:
                    assert np.array_equal(_ints(got, c), want["data"][c][:want["selected"]]), c
                elif c in (6, 7) if name == "pax" else True:
                    ptr, ln = want["data"][c], want["lens"][c]
                    oracle = [bytes(table.image[int(o):int(o) + int(k)]) for o, k in zip(ptr[:want["selected"]], ln[:want["selected"]])]
                    got_c = [b"" if s is None else s for s in _strings(got, c)]
                    assert got_c == oracle, c
    finally:
        p.close()


def test_stored_pipeline_with_skip_index(ob):
    from oceanbase_b200.pipeline import HostScanPipeline
    from oceanbase_b200.sstable import compress_table
    rng = np.random.default_rng(8)
    n, rpb = 40_000, 500
    k = np.sort(rng.integers(0, 1 << 30, size=n, dtype=np.int64))
    v = rng.integers(0, 100, size=n, dtype=np.int64)
    s = [b"v%02d" % x for x in v]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_INTEGER_BASE_DIFF, k), ob.Column(ob.OBJ_INT, ob.ENC_RAW, v), ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s)]
    table = ob.encode_table(cols, rpb)
    rows, offs = ob.table_agg_rows(cols, [0, 1], rpb)
    flt = ob.And([ob.White(0, ob.WHITE_OP_BT, (int(k[9_000]), int(k[21_000]))), ob.White(1, ob.WHITE_OP_LT, (60,))])
    p = HostScanPipeline(0, n_workers=3)
    try:
        plain = p.scan(table, flt, [0, 1, 2], blocks_per_batch=9, selectivity_hint=0.3, ramp=2, agg_rows=rows, agg_off=offs,
                       aggs=[(ob.AGG_SUM, 1, -1)], heap_bytes=0)
        for comp in (2, 4, 6):
            got = p.scan(compress_table(table, comp), flt, [0, 1, 2], blocks_per_batch=9, selectivity_hint=0.3, ramp=2, agg_rows=rows,
                         agg_off=offs, aggs=[(ob.AGG_SUM, 1, -1)], compressor=comp)
            _same(plain, got, [False, False, True])
        want = ora.scan_table(table, flt, [0, 1], [False, False], [8, 8])
        assert plain.selected_rows == want["selected"]
    finally:
        p.close()


def test_heap_mode_on_plain_images(ob, tables, pipe):
    table, vals, nulls, str_cols = tables["pax"]
    flt = _filter(ob, "pax")
    ordinary = [0, 1, 6, 7]
    base = table.image.ctypes.data
    ptr_mode = pipe.scan(table, flt, ordinary, blocks_per_batch=5, selectivity_hint=0.1, string_base=base)
    heap_mode = pipe.scan(table, flt, ordinary, blocks_per_batch=5, selectivity_hint=0.1, heap_bytes=0)
    assert ptr_mode.batches[0].sources[2][0] is table.image and heap_mode.batches[0].sources[2][0] is not table.image
    _same(ptr_mode, heap_mode, [False, False, True, True])
    assert heap_mode.d2h_bytes > ptr_mode.d2h_bytes
    # rebuilt columns: refused without a heap, equal to obgpu_result_fetch_strings of one batch with one
    rebuilt = [0, 8, 9, 10]
    with pytest.raises(ob.ObGpuError) as e:
        pipe.scan(table, flt, rebuilt, blocks_per_batch=5, selectivity_hint=0.1)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    out = pipe.scan(table, flt, rebuilt, blocks_per_batch=5, selectivity_hint=0.1, heap_bytes=0)
    ctx = ob.ScanContext(0)
    batch = ctx.open_batch(table)
    res = batch.scan(flt, rebuilt)
    assert res.selected_rows == out.selected_rows
    for c in (1, 2, 3):
        heap, off = res.fetch_strings(c)
        _, _, nw = res.fetch_col(c)
        want = [None if (int(nw[k >> 6]) >> (k & 63)) & 1 else bytes(heap[off[k]:off[k + 1]]) for k in range(res.selected_rows)]
        assert _strings(out, c) == want, c
    res.free()
    batch.close()
    ctx.close()


def _heap_calls(ob, res, cols, row_begin, rows):
    from oceanbase_b200.capi import lib
    n = len(cols)
    ca = (C.c_int32 * n)(*cols)
    nbytes = np.zeros(n, dtype=np.int64)
    code = lib.obgpu_result_string_bytes(res._h, n, ca, row_begin, rows, nbytes.ctypes.data)
    if code:
        return code, None
    heaps = [np.zeros(max(int(b), 1), dtype=np.uint8) for b in nbytes]
    ptrs = [np.zeros(max(rows, 1), dtype=np.uint64) for _ in cols]
    hh = (C.c_void_p * n)(*[h.ctypes.data for h in heaps])
    hp = (C.c_void_p * n)(*[p.ctypes.data for p in ptrs])
    code = lib.obgpu_result_fetch_string_heap(res._h, n, ca, row_begin, rows, hh, hp)
    if code:
        return code, None
    lens = [res.fetch_col(c, row_begin, rows)[1] for c in cols]
    nws = [res.fetch_col(c, row_begin, rows)[2] for c in cols]
    cells = []
    for j in range(n):
        col = []
        for k in range(rows):
            p = int(ptrs[j][k])
            if (int(nws[j][k >> 6]) >> (k & 63)) & 1:
                assert p == 0
                col.append(None)
            else:
                o = p - heaps[j].ctypes.data
                assert 0 <= o <= nbytes[j]
                col.append(heaps[j][o:o + int(lens[j][k])].tobytes())
        assert sum(len(x) for x in col if x is not None) == nbytes[j]
        cells.append(col)
    return 0, cells


def test_string_heap_calls_directly(ob, tables):
    from oceanbase_b200.capi import lib
    table, vals, nulls, str_cols = tables["pax"]
    ctx = ob.ScanContext(0)
    batch = ctx.open_batch(table)
    proj = [0, 6, 7, 8, 10]   # empty strings and NULL rows in 6, rebuilt columns 8 and 10
    res = batch.scan(_filter(ob, "pax"), proj)
    sel = res.selected_rows
    assert sel > 1000
    for cols, rb, rows in (([1, 2, 3, 4], 0, sel), ([4, 1], 37, 500), ([2], sel - 3, 3), ([1, 3], 0, 0)):
        code, cells = _heap_calls(ob, res, cols, rb, rows)
        assert code == 0
        for j, c in enumerate(cols):
            heap, off = res.fetch_strings(c, rb, rows)
            _, _, nw = res.fetch_col(c, rb, rows)
            want = [None if (int(nw[k >> 6]) >> (k & 63)) & 1 else bytes(heap[off[k]:off[k + 1]]) for k in range(rows)]
            assert cells[j] == want, (cols, c)
    assert any(s == b"" for s in _heap_calls(ob, res, [1], 0, sel)[1][0])
    r = batch.scan(ob.White(7, ob.WHITE_OP_NE, (b"w003",)), proj)   # NULL rows of column 6 pass this filter
    assert any(s is None for s in _heap_calls(ob, r, [1], 0, r.selected_rows)[1][0])
    r.free()
    # the fetch must name the rows and columns the size call sized
    ca = (C.c_int32 * 2)(1, 2)
    nb = np.zeros(2, dtype=np.int64)
    assert lib.obgpu_result_string_bytes(res._h, 2, ca, 5, 100, nb.ctypes.data) == 0
    heaps = [np.zeros(int(b) + 1, dtype=np.uint8) for b in nb]
    hh = (C.c_void_p * 2)(*[h.ctypes.data for h in heaps])
    for cols, rb, rows in (([2, 1], 5, 100), ([1, 2], 6, 100), ([1, 2], 5, 99), ([1], 5, 100)):
        cb = (C.c_int32 * len(cols))(*cols)
        assert lib.obgpu_result_fetch_string_heap(res._h, len(cols), cb, rb, rows, hh, None) == ob.OB_INVALID_ARGUMENT
    assert lib.obgpu_result_fetch_string_heap(res._h, 2, ca, 5, 100, hh, None) == 0
    assert lib.obgpu_result_string_bytes(res._h, 1, (C.c_int32 * 1)(0), 0, 10, nb.ctypes.data) == ob.OB_INVALID_ARGUMENT  # integer column
    assert lib.obgpu_result_string_bytes(res._h, 1, (C.c_int32 * 1)(1), 0, sel + 1, nb.ctypes.data) == ob.OB_INVALID_ARGUMENT
    # the result object stays consistent: fetch_cols / fetch_strings answer as before
    d0, _, n0 = res.fetch_col(0)
    want = ora.scan_table(table, _filter(ob, "pax"), [0], [False], [8])
    assert np.array_equal(d0, want["data"][0][:sel])
    # launch counts: the same for different selected rows and for one or three columns
    counts = []
    for flt in (_filter(ob, "pax"), ob.White(1, ob.WHITE_OP_LT, (5,))):
        r = batch.scan(flt, proj)
        for cols in ([1], [1, 2, 4]):
            c0 = ctx.launch_count
            code, _ = _heap_calls(ob, r, cols, 0, r.selected_rows)
            assert code == 0
            counts.append(ctx.launch_count - c0)
        r.free()
    assert len(set(counts)) == 1 and counts[0] > 0, counts
    res.free()
    batch.close()
    ctx.close()


def test_errors_leave_the_pipeline_usable(ob, tables):
    from oceanbase_b200 import capi
    from oceanbase_b200.pipeline import HostOutputs, HostScanPipeline
    from oceanbase_b200.sstable import compress_table
    table, vals, nulls, str_cols = tables["cs"]
    stored = compress_table(table, 6)
    proj = [0, 1, 4, 5]
    p = HostScanPipeline(0, n_workers=3)
    good = p.scan(stored, None, proj, blocks_per_batch=6, selectivity_hint=1.0, compressor=6)

    def again():
        out = p.scan(stored, None, proj, blocks_per_batch=6, selectivity_hint=1.0, compressor=6)
        _same(good, out, [False, False, True, True])

    def code_of(fn):
        with pytest.raises(capi.ObGpuError) as e:
            fn()
        return e.value.code, str(e.value)

    # a string column of compressed blocks without a heap: refused, and the message names the column
    outs = HostOutputs.allocate(table.total_rows + 4096, [False, False, True, True], [8, 8, 8, 8])
    code, msg = code_of(lambda: p.scan(stored, None, proj, 6, 1.0, outputs=outs, compressor=6))
    assert code == capi.OB_NOT_SUPPORTED and "column 2" in msg
    again()
    # a heap too small: OBGPU_BUF_NOT_ENOUGH naming the column; then success with the reported size
    outs = HostOutputs.allocate(table.total_rows + 4096, [False, False, True, True], [8, 8, 8, 8], heap_bytes=1000)
    code, msg = code_of(lambda: p.scan(stored, None, proj, 6, 1.0, outputs=outs, compressor=6))
    assert code == capi.OB_BUF_NOT_ENOUGH and "column" in msg
    need = sum(len(s) for s in _strings(good, 2) if s) + sum(len(s) for s in _strings(good, 3) if s)
    outs = HostOutputs.allocate(table.total_rows + 4096, [False, False, True, True], [8, 8, 8, 8], heap_bytes=need)
    _same(good, p.scan(stored, None, proj, 6, 1.0, outputs=outs, compressor=6), [False, False, True, True])
    # the Python entry grows its own heaps: a tiny first size still succeeds
    _same(good, p.scan(stored, None, proj, 6, 1.0, compressor=6, heap_bytes=64), [False, False, True, True])
    # zero copy with a compressor, unknown compressors
    code, msg = code_of(lambda: p.scan(stored, None, [0, 1], 6, 1.0, compressor=6, zero_copy=True))
    assert code == capi.OB_NOT_SUPPORTED
    again()
    for comp in (3, 5, 11, -1):
        code, msg = code_of(lambda: p.scan(stored, None, [0, 1], 6, 1.0, outputs=HostOutputs.allocate(table.total_rows + 4096, [False, False], [8, 8]),
                                           compressor=comp))
        assert code == capi.OB_NOT_SUPPORTED, comp
        again()
    # one corrupt block in a middle batch: OBGPU_INVALID_DATA from the open
    bad = stored.image.copy()
    mid = stored.n_blocks // 2
    o = int(stored.offsets[mid])
    bad[o + int(stored.sizes[mid]) - 3] ^= 0x5A
    from oceanbase_b200.sstable import TableImage
    broken = TableImage(bad, stored.offsets, stored.sizes, stored.total_rows, stored.n_cols)
    code, msg = code_of(lambda: p.scan(broken, None, proj, 6, 1.0, compressor=6))
    assert code == capi.OB_INVALID_DATA
    again()
    # no_row_output needs no heap
    agg = p.scan(stored, None, [0, 1, 4], 6, 1.0, compressor=6, no_row_output=True, aggs=[(ob.AGG_COUNT, 1, -1)])
    assert agg.aggregates[0] == int(np.count_nonzero(nulls[1] == 0))
    p.close()
