"""The device group accumulator (obgpu_groups_*, ScanContext.group_accumulator) against a plain tuple model of the generator's
cells (test_gpu_group_by_columns.tuple_model) and, byte for byte, against obgpu_result_group_by_columns over the same rows opened
as one batch. Every table is cut into page batches by block; each batch is opened, scanned, grouped, added, and its result freed
and batch closed at once, so the accumulator never reads a batch after its add.

Cases: 1. every integer type x codec of the aggregate matrix; 2. PAX, CS and mixed batches, dictionaries that differ between
batches for the same values; 3. strings, also from LZ4- and zstd-stored batches; 4. NULL in several columns; 5. every order of
the adds of four batches, and adds from a second ctx; 6. 128-bit SUM carries across adds, unsigned 64-bit and signed MIN / MAX
extremes, a MIN that is NULL-only in one batch; 7. growth at both sides of each rebuild of the table, and of the string key heap
past 64 and 128 KiB; 8. refusals, with the fetch unchanged after each; 9. zero groups."""
import ctypes as C
import itertools

import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM, MATRIX, K, matrix_spec, matrix_table
from test_gpu_aggregate_exact import GROUP_AGGS
from test_gpu_group_by_columns import tuple_model
from test_scan_codes_model import concat_table, cs_table, open_table, string_table, CS_MODES

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx2(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def cut(table, bounds):
    """the page batches of blocks [bounds[i], bounds[i + 1]) as tables of their own"""
    from oceanbase_b200.sstable import TableImage
    n = table.n_blocks
    parts = []
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        lo = int(table.offsets[b0])
        hi = int(table.offsets[b1]) if b1 < n else int(table.image.size)
        parts.append(TableImage(np.ascontiguousarray(table.image[lo:hi]), table.offsets[b0:b1] - lo, table.sizes[b0:b1], 0, table.n_cols))
    return parts


def raw_groups(ob, res, gcols, aggs):
    """obgpu_result_group_by_columns + obgpu_result_fetch_group_columns: (keys, nulls, heap, out) as fetched"""
    lib = ob.capi.lib
    g = np.array(gcols, dtype=np.int32)
    spec = np.array(aggs, dtype=np.int32).reshape(-1, 2)
    ng, kb = C.c_int64(), C.c_int64()
    ob.capi.check(lib.obgpu_result_group_by_columns(res._h, g.ctypes.data, len(gcols), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb)),
                  "obgpu_result_group_by_columns", res.batch.ctx._h)
    n = ng.value
    keys = np.zeros((len(gcols), n + 1), dtype=np.int64)
    nulls = np.zeros((len(gcols), max(n, 1)), dtype=np.uint8)
    heap = np.zeros(max(kb.value, 1), dtype=np.uint8)
    out = np.zeros((len(aggs), max(n, 1), 2), dtype=np.int64)
    ob.capi.check(lib.obgpu_result_fetch_group_columns(res._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data),
                  "obgpu_result_fetch_group_columns", res.batch.ctx._h)
    return keys, nulls[:, :n], heap[:kb.value], out[:, :n]


def same_bytes(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def add_parts(ob, acc, ctxs, parts, gcols, aggs, flt=None, order=None, compressor=None):
    """each part opened on ctxs[i % len(ctxs)], scanned, grouped and added; its result freed and its batch closed right after"""
    for i in (range(len(parts)) if order is None else order):
        batch = ctxs[i % len(ctxs)].open_batch(parts[i], compressor=compressor)
        res = batch.scan(flt, [0])
        raw_groups(ob, res, gcols, aggs)
        acc.add(res)
        res.free()
        batch.close()


def one_batch(ob, ctx, table, gcols, aggs, flt=None, compressor=None):
    batch = ctx.open_batch(table, compressor=compressor)
    res = batch.scan(flt, [0])
    raw = raw_groups(ob, res, gcols, aggs)
    res.free()
    batch.close()
    return raw


def check(ob, ctx, table, bounds, gcols, aggs, cells, rows, flt=None, ctxs=None, what=""):
    """the accumulator over the cut equals the tuple model and the one-batch call byte for byte; returns its fetched bytes"""
    acc = ctx.group_accumulator(len(gcols), aggs)
    add_parts(ob, acc, ctxs or [ctx], cut(table, bounds), gcols, aggs, flt)
    keys, out = acc.fetch()
    want_keys, want = tuple_model([cells[c] for c in gcols], list(rows), aggs, cells)
    assert keys == want_keys, what
    assert np.array_equal(out, want), what
    raw = acc.fetch_raw()
    assert same_bytes(raw, one_batch(ob, ctx, table, gcols, aggs, flt)), what
    acc.free()
    return raw


def thirds(n_blocks):
    return sorted({0, n_blocks // 3, 2 * n_blocks // 3, n_blocks})


# ---- 1. every integer type x codec --------------------------------------------------------------------------------------
@pytest.mark.parametrize("tname,codec", MATRIX)
def test_matrix(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    table = matrix_table(tname, codec)
    gcs = list(spec.group_cols.values())
    rows = range(spec.n)
    for gcols in ([gcs[0], gcs[1]], gcs[::-1][:2], [gcs[-1]]):
        check(ob, ctx, table, thirds(table.n_blocks), gcols, GROUP_AGGS, spec.truth, rows, what=gcols)
    sel = [i for i in rows if spec.truth[K][i] < spec.n // 2]
    check(ob, ctx, table, [0, 1, table.n_blocks], gcs[:2], GROUP_AGGS, spec.truth, sel, flt=ob.White(K, ob.WHITE_OP_LT, (spec.n // 2,)))


# ---- 2. PAX, CS, mixed; dictionaries that differ between batches ----------------------------------------------------------
AGGS = [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (COUNT, 1)]


@pytest.mark.parametrize("mode", CS_MODES)
def test_cs_batches(ob, ctx, mode):
    t = cs_table(mode)
    for gcols in ([1, 2], [4, 1, 2]):
        check(ob, ctx, t.image, thirds(t.image.n_blocks), gcols, AGGS, t.cells, range(t.n), what=gcols)


def test_pax_and_cs_batches(ob, ctx):
    t = concat_table()
    n = t.image.n_blocks
    for bounds in (thirds(n), list(range(n + 1))):   # PAX-only, CS-only and mixed batches; one block each
        check(ob, ctx, t.image, bounds, [2, 3, 4], AGGS, t.cells, range(t.n), what=bounds)


def test_dictionaries_differ_between_batches(ob, ctx):
    t = open_table()    # 1 INT DICT over every layout, 2 VARCHAR DICT, 3 UINT64 DICT over every layout
    aggs = [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (SUM, 3)]
    for gcols in ([1, 3], [3, 2, 1]):
        check(ob, ctx, t.image, list(range(t.image.n_blocks + 1)), gcols, aggs, t.cells, range(t.n), what=gcols)


# ---- 3. strings, also from stored blocks closed before the fetch ----------------------------------------------------------
STR_AGGS = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 4), (COUNT, 4)]


def test_strings(ob, ctx):
    t = string_table()
    for gcols in ([1, 2], [2, 1], [2, 4, 1]):
        check(ob, ctx, t.image, thirds(t.image.n_blocks), gcols, STR_AGGS, t.cells, range(t.n), what=gcols)


@pytest.mark.parametrize("comp", ["lz4", "zstd"])
def test_strings_from_stored_blocks(ob, ctx, comp):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    c = {"lz4": ob.capi.COMPRESSOR_LZ4, "zstd": ob.capi.COMPRESSOR_ZSTD_1_3_8}[comp]
    stored = compress_table(t.image, c)
    acc = ctx.group_accumulator(2, STR_AGGS)
    add_parts(ob, acc, [ctx], cut(stored, thirds(stored.n_blocks)), [2, 1], STR_AGGS, compressor=c)   # every batch closed
    keys, out = acc.fetch()
    want_keys, want = tuple_model([t.cells[2], t.cells[1]], list(range(t.n)), STR_AGGS, t.cells)
    assert keys == want_keys and np.array_equal(out, want)
    assert same_bytes(acc.fetch_raw(), one_batch(ob, ctx, t.image, [2, 1], STR_AGGS))
    acc.free()


# ---- 4. NULL in several columns -------------------------------------------------------------------------------------------
def nulls_table(ob, n=3000, seed=23):
    rng = np.random.default_rng(seed)
    a = [int(x) for x in rng.integers(-3, 4, n)]
    s = [b"k%d" % int(x) for x in rng.integers(0, 5, n)]
    za, zs = rng.random(n) < 0.2, rng.random(n) < 0.2
    w = [int(x) for x in rng.integers(-1000, 1000, n)]
    cols = [ob.Column(5, 0, np.arange(n, dtype=np.int64)), ob.Column(5, 1, np.array(a, dtype=np.int64), nulls=za.astype(np.uint8)),
            ob.Column(22, 1, s, nulls=zs.astype(np.uint8)), ob.Column(5, 0, np.array(w, dtype=np.int64))]
    cells = [list(range(n)), [None if z else v for v, z in zip(a, za)], [None if z else v for v, z in zip(s, zs)], w]
    return ob.encode_table(cols, 133), cells


def test_nulls_in_several_columns(ob, ctx):
    table, cells = nulls_table(ob)
    aggs = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 3), (COUNT, 1)]
    n = len(cells[0])
    for gcols in ([1, 2], [2, 1], [2, 1, 2, 1]):
        check(ob, ctx, table, thirds(table.n_blocks), gcols, aggs, cells, range(n), what=gcols)
    keys, _ = ctx.group_accumulator(2, aggs).fetch()
    assert keys == []


# ---- 5. every order of the adds; a second ctx ----------------------------------------------------------------------------
def test_every_add_order_gives_the_same_bytes(ob, ctx, ctx2):
    table, cells = nulls_table(ob)
    aggs = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 3)]
    n = table.n_blocks
    parts = cut(table, [0, 3, n // 2, n - 2, n])
    first = None
    for order in itertools.permutations(range(4)):
        acc = ctx.group_accumulator(2, aggs)
        add_parts(ob, acc, [ctx, ctx2], parts, [2, 1], aggs, order=order)
        raw = acc.fetch_raw()
        acc.free()
        first = raw if first is None else first
        assert same_bytes(raw, first), order
    assert same_bytes(first, one_batch(ob, ctx, table, [2, 1], aggs))


def test_adds_from_a_second_ctx(ob, ctx, ctx2):
    t = string_table()
    check(ob, ctx, t.image, thirds(t.image.n_blocks), [1, 2], STR_AGGS, t.cells, range(t.n), ctxs=[ctx2])
    check(ob, ctx, t.image, list(range(t.image.n_blocks + 1)), [2, 1], STR_AGGS, t.cells, range(t.n), ctxs=[ctx, ctx2])


# ---- 6. carries and extremes across adds ----------------------------------------------------------------------------------
def extremes_table(ob):
    """0 row id; 1 INT DICT key 0..3; 2 UINT64 near 2^64 and at 0 / 2^63; 3 INT64 at both ends; 4 INT with a NULL-only block"""
    n, rpb = 1600, 100
    i = np.arange(n)
    key = (i % 4).astype(np.int64)
    u = np.array([U64_MAX - (x % 7) if x % 5 else [0, 1 << 63, U64_MAX][x % 3] for x in range(n)], dtype=np.uint64)
    s = np.array([[I64_MIN, I64_MAX, I64_MIN + 1, -1][x % 4] if x % 3 else I64_MIN for x in range(n)], dtype=np.int64)
    v = (i * 37 % 1000 - 500).astype(np.int64)
    zv = ((i // rpb) % 2 == 0).astype(np.uint8)          # even blocks: every cell NULL
    zv[(i // rpb) % 2 == 1] = (i[(i // rpb) % 2 == 1] % 9 == 0)
    cols = [ob.Column(5, 0, i.astype(np.int64)), ob.Column(5, 1, key), ob.Column(10, 0, u.view(np.int64)),
            ob.Column(5, 0, s), ob.Column(5, 0, v, nulls=zv)]
    cells = [i.tolist(), key.tolist(), [int(x) for x in u.tolist()], s.tolist(), [None if z else int(x) for x, z in zip(v.tolist(), zv)]]
    return ob.encode_table(cols, rpb), cells


def test_carries_and_extremes_across_adds(ob, ctx):
    table, cells = extremes_table(ob)
    aggs = [(COUNT, -1), (SUM, 2), (SUM, 3), (MIN, 2), (MAX, 2), (MIN, 3), (MAX, 3), (MIN, 4), (MAX, 4), (COUNT, 4), (SUM, 4)]
    n = table.n_blocks
    raw = check(ob, ctx, table, list(range(n + 1)), [1], aggs, cells, range(len(cells[0])))
    out = raw[3]
    assert (out[1, :, 1] > 1).all() and (out[2, :, 1] != 0).all()                    # 128-bit sums that carried across adds
    assert out[3, :, 0].tolist() == [0] * 4 and out[4, :, 0].tolist() == [-1] * 4    # UINT64 MIN 0, MAX 2^64 - 1
    assert out[5, :, 0].tolist() == [I64_MIN] * 4 and I64_MAX in out[6, :, 0].tolist()
    # a group whose MIN / MAX is NULL-only in every even batch: the odd batches' values are what come back
    acc = ctx.group_accumulator(1, [(MIN, 4), (MAX, 4)])
    add_parts(ob, acc, [ctx], cut(table, list(range(n + 1))), [1], [(MIN, 4), (MAX, 4)], order=[0, 2, 4, 1, 3, 5, 6, 7, 8])
    _, got = acc.fetch()
    rows = [r for r in range(len(cells[0])) if r < 900]
    _, want = tuple_model([cells[1]], rows, [(MIN, 4), (MAX, 4)], cells)
    assert np.array_equal(got, want) and (got[:, :, 1] == 1).all()
    acc.free()


# ---- 7. growth at both sides of each rebuild ------------------------------------------------------------------------------
INIT_GROUPS = 1024


def keyed_table(ob, keys, row0=0):
    n = len(keys)
    k = np.asarray(keys, dtype=np.int64)
    return ob.encode_table([ob.Column(5, 0, np.arange(row0, row0 + n, dtype=np.int64)), ob.Column(5, 1, k),
                            ob.Column(5, 0, k * 3 - 7)], 256)


# (groups of the batch, of them new): the accumulator's capacity is 1024 and doubles when its groups plus a batch's exceed it
GROWTH = [("1023 new: capacity 1024", list(range(1023))),
          ("1 new: 1024 groups, at capacity", [5000]),
          ("1 old: 1025 > 1024, rebuilt at 2048", [7]),
          ("1024 new: 2048, at capacity", list(range(10_000, 11_024))),
          ("2 old, 1 new: 2051 > 2048, rebuilt at 4096", [3, 10_500, 20_000]),
          ("old and new mixed", list(range(0, 40_000, 13)))]


def test_growth_at_both_sides_of_each_rebuild(ob, ctx):
    aggs = [(COUNT, -1), (SUM, 2), (MIN, 2), (MAX, 2)]
    acc = ctx.group_accumulator(1, aggs)
    all_keys, row0 = [], 0
    for what, keys in GROWTH:
        keys = keys * 2     # every key twice per batch
        batch = ctx.open_batch(keyed_table(ob, keys, row0))
        res = batch.scan(None, [0])
        res.group_by_columns([1], aggs)
        acc.add(res)
        res.free()
        batch.close()
        all_keys += keys
        row0 += len(keys)
        cells = [list(range(row0)), all_keys, [k * 3 - 7 for k in all_keys]]
        got_keys, got = acc.fetch()
        want_keys, want = tuple_model([all_keys], list(range(row0)), aggs, cells)
        assert got_keys == want_keys and np.array_equal(got, want), what
    assert same_bytes(acc.fetch_raw(), one_batch(ob, ctx, keyed_table(ob, all_keys), [1], aggs))
    acc.free()


def str_keyed_table(ob, keys, row0=0):
    n = len(keys)
    return ob.encode_table([ob.Column(5, 0, np.arange(row0, row0 + n, dtype=np.int64)), ob.Column(22, 1, list(keys)),
                            ob.Column(5, 0, np.arange(row0, row0 + n, dtype=np.int64) % 97 - 40)], 64)


def key200(k):
    return b"%05d" % k + bytes([0x41 + k % 26]) * 195


# (key bytes of the accumulator after the add): the key heap starts at 64 KiB and doubles when its bytes plus a result's exceed it
HEAP_GROWTH = [("320 keys: 64 000 B, in the first 64 KiB", list(range(320)), 64_000),
               ("8 new, 8 old: 64 000 + 3 200 > 65 536, grown to 128 KiB", list(range(312, 328)), 65_600),
               ("330 new: 65 600 + 66 000 > 131 072, grown to 256 KiB", list(range(1000, 1330)), 131_600),
               ("old keys only: no new bytes", list(range(0, 328, 3)) + list(range(1000, 1330, 5)), 131_600)]


def test_key_heap_grows_past_64_and_128_kib(ob, ctx):
    aggs = [(COUNT, -1), (SUM, 2), (MIN, 2)]
    acc = ctx.group_accumulator(1, aggs)
    all_keys, row0 = [], 0
    for what, ks, heap_bytes in HEAP_GROWTH:
        keys = [key200(k) for k in ks]
        batch = ctx.open_batch(str_keyed_table(ob, keys, row0))
        res = batch.scan(None, [0])
        res.group_by_columns([1], aggs)
        acc.add(res)
        res.free()
        batch.close()
        all_keys += keys
        row0 += len(keys)
        assert acc.info()[1] == heap_bytes, what
        cells = [list(range(row0)), all_keys, [r % 97 - 40 for r in range(row0)]]
        got_keys, got = acc.fetch()
        want_keys, want = tuple_model([all_keys], list(range(row0)), aggs, cells)
        assert got_keys == want_keys and np.array_equal(got, want), what
    assert same_bytes(acc.fetch_raw(), one_batch(ob, ctx, str_keyed_table(ob, all_keys), [1], aggs))
    acc.free()


# ---- 8. refusals leave the accumulator as it was --------------------------------------------------------------------------
def test_refusals(ob, ctx):
    table, cells = nulls_table(ob)
    aggs = [(COUNT, -1), (SUM, 3), (MIN, 3)]
    parts = cut(table, thirds(table.n_blocks))
    acc = ctx.group_accumulator(2, aggs)
    add_parts(ob, acc, [ctx], parts[:1], [1, 2], aggs)
    before = acc.fetch_raw()
    other, _ = nulls_table(ob, n=500, seed=5)
    typed = ob.encode_table([ob.Column(5, 0, np.arange(500, dtype=np.int64)), ob.Column(4, 1, np.arange(500, dtype=np.int64) % 3),
                             ob.Column(22, 1, [b"x"] * 500), ob.Column(5, 0, np.arange(500, dtype=np.int64))], 133)
    agg_typed = ob.encode_table([ob.Column(5, 0, np.arange(500, dtype=np.int64)), ob.Column(5, 1, np.arange(500, dtype=np.int64) % 3),
                                 ob.Column(22, 1, [b"x"] * 500), ob.Column(4, 0, np.arange(500, dtype=np.int64))], 133)
    cases = [("one group column", other, [1], aggs), ("three group columns", other, [1, 2, 1], aggs),
             ("another kind", other, [1, 2], [(COUNT, -1), (SUM, 3), (MAX, 3)]),
             ("another column", other, [1, 2], [(COUNT, -1), (SUM, 0), (MIN, 3)]),
             ("fewer aggregates", other, [1, 2], aggs[:2]),
             ("group column type", typed, [1, 2], aggs), ("aggregate column type", agg_typed, [1, 2], aggs)]
    for what, t, gcols, ag in cases:
        batch = ctx.open_batch(t)
        res = batch.scan(None, [0])
        res.group_by_columns(gcols, ag)
        with pytest.raises(ob.ObGpuError) as e:
            acc.add(res)
        assert e.value.code == ob.OB_NOT_SUPPORTED, what
        res.free()
        batch.close()
        assert same_bytes(acc.fetch_raw(), before), what
    batch = ctx.open_batch(other)
    res = batch.scan(None, [0])
    with pytest.raises(ob.ObGpuError) as e:      # no groups on the result
        acc.add(res)
    assert e.value.code == ob.OB_INVALID_ARGUMENT
    res.group_by_columns([1], aggs)
    try:
        res.group_by_columns([1, 3], aggs)       # a refused call leaves the result with no groups
    except ob.ObGpuError:
        pass
    with pytest.raises(ob.ObGpuError) as e:
        acc.add(res)
    assert e.value.code == ob.OB_INVALID_ARGUMENT
    res.free()
    batch.close()
    assert same_bytes(acc.fetch_raw(), before)
    add_parts(ob, acc, [ctx], parts[1:], [1, 2], aggs)     # still usable: the rest of the table
    keys, out = acc.fetch()
    want_keys, want = tuple_model([cells[1], cells[2]], list(range(len(cells[0]))), aggs, cells)
    assert keys == want_keys and np.array_equal(out, want)
    lib = ob.capi.lib
    spec = np.array(aggs, dtype=np.int32)
    h = C.c_void_p()
    for n_cols, n_aggs in ((0, 3), (5, 3), (2, 0), (2, 17)):
        assert lib.obgpu_groups_create(ctx._h, n_cols, spec.ctypes.data, n_aggs, C.byref(h)) == ob.OB_INVALID_ARGUMENT
    acc.free()


# ---- 9. zero groups -------------------------------------------------------------------------------------------------------
def test_zero_groups(ob, ctx):
    table, cells = nulls_table(ob)
    aggs = [(COUNT, -1), (SUM, 3)]
    acc = ctx.group_accumulator(2, aggs)
    assert acc.info() == (0, 0, [(0, -1), (0, -1)])
    empty = acc.fetch_raw()
    keys, out = acc.fetch()
    assert keys == [] and out.shape == (2, 0, 2)
    add_parts(ob, acc, [ctx], cut(table, thirds(table.n_blocks)), [1, 2], aggs, flt=ob.White(0, ob.WHITE_OP_LT, (0,)))
    keys, out = acc.fetch()
    assert keys == [] and out.shape == (2, 0, 2)
    assert same_bytes(acc.fetch_raw(), empty)
    assert same_bytes(empty, one_batch(ob, ctx, table, [1, 2], aggs, flt=ob.White(0, ob.WHITE_OP_LT, (0,))))
    assert acc.info()[2] == [(5, 8), (22, 0)]
    acc.free()
