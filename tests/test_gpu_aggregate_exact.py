"""Pushed-down aggregates and GROUP BY on the device against exact Python integer folds (tests/test_aggregate_exact.py):
every integer type at its extremes, every value codec (PAX RAW bit-packed / byte-packed / with NULLs, DICT, RLE, CONST with
and without exceptions, INTEGER_BASE_DIFF, CS INTEGER, CS INT_DICT), every entry point that folds them --
obgpu_result_aggregate, obgpu_block_group_by, obgpu_result_group_by on every count-kernel path (pipelined kernels on and
off, lean and general kernels, skip-index settled blocks, a capacity-overflowed scan) and the host pipeline's per-batch fold.
Every comparison is exact."""
import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import (COUNT, SUM, SUM_PRODUCT, MIN, MAX, TYPES, MATRIX, K, M, W, VA, VB, VN, M64, matrix_spec, matrix_table, block_cells, fold, exact_group_by_model, gen_values, as_store,
                                  with_nulls, to_i64)

pytestmark = pytest.mark.gpu

PROJ = [K, M, W, VA, VB, VN]          # projection index == store column
PAIRS = [(VA, W), (VB, W), (VA, VB), (W, W), (VN, W)]
GROUP_AGGS = [(COUNT, -1), (COUNT, VA), (COUNT, VB), (SUM, VA), (SUM, VB), (MIN, VA), (MAX, VA), (MIN, VB), (MAX, VB),
              (SUM, VN), (MIN, VN), (MAX, VN), (COUNT, VN), (SUM, W), (MIN, W), (MAX, W)]


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def check_aggregates(res, truth, rows, what):
    """every aggregate kind over the projected columns of `res` (projection index == index into truth) vs the fold"""
    assert res.selected_rows == len(rows), what
    cells = {c: [truth[c][i] for i in rows] for c in (W, VA, VB, VN)}
    for c in (W, VA, VB, VN):
        for kind in (COUNT, SUM, MIN, MAX):
            assert res.aggregate(kind, c) == fold(kind, cells[c]), (what, kind, c)
    for a, b in PAIRS:
        assert res.aggregate(SUM_PRODUCT, a, b) == fold(SUM_PRODUCT, cells[a], cells[b]), (what, a, b)


@pytest.mark.parametrize("tname,codec", MATRIX)
def test_result_aggregate(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    table = matrix_table(tname, codec)
    _, lo, hi = TYPES[tname]
    va, vb, m = spec.truth[VA], spec.truth[VB], spec.truth[M]
    n = spec.n
    i_max = next((i for i, x in enumerate(va) if x == hi), 0)     # a single row holding the type's maximum / minimum:
    i_min = next((i for i, x in enumerate(va) if x == lo), 1)     # MIN / MAX equal to the fold's initial key for INT, UINT64
    cases = [
        ("no filter", None, range(n)),
        ("every row", ob.White(K, ob.WHITE_OP_GE, (0,)), range(n)),
        ("one row (max)", ob.White(K, ob.WHITE_OP_EQ, (i_max,)), [i_max]),
        ("one row (min)", ob.White(K, ob.WHITE_OP_EQ, (i_min,)), [i_min]),
        ("no row", ob.White(K, ob.WHITE_OP_LT, (0,)), []),
        ("sparse", ob.White(M, ob.WHITE_OP_LT, (3,)), [i for i in range(n) if m[i] < 3]),
        ("VB NULL", ob.White(VB, ob.WHITE_OP_NU, ()), [i for i in range(n) if vb[i] is None]),
    ]
    batch = ctx.open_batch(table)
    for what, flt, rows in cases:
        res = batch.scan(flt, PROJ)
        check_aggregates(res, spec.truth, list(rows), what)
        if what == "VB NULL":        # every selected row NULL in VB
            assert res.aggregate(MIN, VB) is None and res.aggregate(MAX, VB) is None
            assert res.aggregate(COUNT, VB) == 0 and res.aggregate(SUM, VB) == 0
        res.free()
    # a result that overflowed its capacity has no aggregate: the scan's status comes back instead of a number
    for flt, cap in ((None, n - 1), (ob.White(M, ob.WHITE_OP_LT, (50,)), 10)):
        res = batch.scan(flt, PROJ, max_selected_rows=cap)
        for kind, b in ((SUM, -1), (SUM_PRODUCT, W), (MIN, -1), (COUNT, -1)):
            with pytest.raises(ob.ObGpuError) as e:
                res.aggregate(kind, VA, b)
            assert e.value.code == ob.OB_BUF_NOT_ENOUGH
        res.free()
    batch.close()


@pytest.mark.parametrize("tname,codec", MATRIX)
def test_group_by(ob, ctx, tname, codec):
    spec = matrix_spec(tname, codec)
    table = matrix_table(tname, codec)
    batch = ctx.open_batch(table)
    blocks = [ora.Block(table.block(b)) for b in range(table.n_blocks)]
    cells = [block_cells(spec, b) for b in range(table.n_blocks)]
    for gname, gc in spec.group_cols.items():
        # one block, the reference call shape: every row, odd rows, rows in descending order
        for b, blk in enumerate(blocks):
            n = blk.row_count
            for rows in (np.arange(n), np.arange(1, n, 2), np.arange(n - 1, -1, -1)):
                got = batch.group_by(b, gc, GROUP_AGGS, rows)
                assert np.array_equal(got, exact_group_by_model(blk, gc, rows, GROUP_AGGS, cells[b])), (gname, b, len(rows))
        # every block of a scan, the rows its filter selected
        m = spec.truth[M]
        for flt, keep in ((None, lambda i: True), (ob.White(K, ob.WHITE_OP_GE, (0,)), lambda i: True),
                          (ob.White(M, ob.WHITE_OP_LT, (40,)), lambda i: m[i] < 40)):
            res = batch.scan(flt, [K])
            goff, out = res.group_by(gc, GROUP_AGGS)
            for b, blk in enumerate(blocks):
                r0 = b * spec.rpb
                rows = np.array([r for r in range(blk.row_count) if keep(r0 + r)], dtype=np.int32)
                assert np.array_equal(out[:, goff[b]:goff[b + 1]], exact_group_by_model(blk, gc, rows, GROUP_AGGS, cells[b])), (gname, b)
            res.free()
    batch.close()


# ---- GROUP BY over a scan on every count-kernel path ------------------------------------------------------------------
PATH_TYPES = ["int", "uint64", "date", "year", "tinyint", "uint32"]
PATH_AGGS = [[(COUNT, -1)] + [(k, 5 + j) for j in js for k in (COUNT, SUM, MIN, MAX)] for js in ((0, 1, 2), (3, 4, 5))]
PATH_ROWS = {1: 300, 133: 133 * 45, 1100: 11_000, 2000: 16_000}
_path_cache = {}


def path_table(ob, rpb):
    """c0 row number (sorted: the skip index settles whole blocks), c1 0..99, c2 INT DICT / c3 VARCHAR DICT / c4 INT RLE
    group columns, c5.. one value column per PATH_TYPES with 10 % NULL"""
    if rpb in _path_cache:
        return _path_cache[rpb]
    n = PATH_ROWS[rpb]
    rng = np.random.default_rng(rpb)
    k = list(range(n))
    m = [int(x) for x in rng.integers(0, 100, size=n).tolist()]
    gkey = rng.integers(0, 16, size=n)
    ng = (rng.random(n) < 0.05).astype(np.uint8)
    if rpb == 1:
        ng[:] = 0        # a one-row block whose only cell is NULL cannot be dictionary coded (the writer refuses it)
    gint = [int(g) * 7919 - 60_000 for g in gkey.tolist()]
    words = [b"grp%02d" % i for i in range(16)]
    runs = (np.repeat(rng.integers(0, 6, size=n // 25 + 1), 25)[:n] * 3).tolist()
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, as_store(k)), ob.Column(ob.OBJ_INT, ob.ENC_RAW, as_store(m)),
            ob.Column(ob.OBJ_INT, ob.ENC_DICT, as_store(gint), nulls=ng),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, [words[g] for g in gkey.tolist()], nulls=ng),
            ob.Column(ob.OBJ_INT, ob.ENC_RLE, as_store(runs))]
    truth = [k, m, None, None, None]
    for t in PATH_TYPES:
        v = gen_values(rng, t, "free", n, "hi" if t != "date" else "lo")
        nv = (rng.random(n) < 0.10).astype(np.uint8)
        cols.append(ob.Column(TYPES[t][0], ob.ENC_RAW, as_store(v), nulls=nv))
        truth.append(with_nulls(v, nv))
    table = ob.encode_table(cols, rpb)
    agg = ob.table_agg_rows(cols, [0, 1], rpb)
    blocks = [ora.Block(table.block(b)) for b in range(table.n_blocks)]
    _path_cache[rpb] = (table, agg, truth, blocks)
    return _path_cache[rpb]


@pytest.fixture(params=["1", "0"], ids=["pipe", "no_pipe"])
def pipe(request, monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", request.param)
    return request.param


@pytest.mark.parametrize("rpb", [1, 133, 1100, 2000])
def test_result_group_by_on_every_count_path(ob, ctx, pipe, rpb):
    table, agg, truth, blocks = path_table(ob, rpb)
    n = PATH_ROWS[rpb]
    m = truth[M]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    cases = [
        ("no filter", None, lambda i: True),
        ("every row", ob.White(0, ob.WHITE_OP_GE, (0,)), lambda i: True),
        ("key range", ob.White(0, ob.WHITE_OP_BT, (lo, hi)), lambda i: lo <= i <= hi),
        ("key range and m", ob.And([ob.White(0, ob.WHITE_OP_BT, (lo, hi)), ob.White(1, ob.WHITE_OP_LT, (50,))]),
         lambda i: lo <= i <= hi and m[i] < 50),
    ]
    batch = ctx.open_batch(table)
    for with_index in (False, True):
        batch.set_agg_rows(*agg) if with_index else batch.set_agg_rows(None)
        for what, flt, keep in cases:
            res = batch.scan(flt, [0])
            if with_index and what == "key range":
                never, always = res.skip_info()
                assert never > 0 and always > 0, (never, always)
            sel = [np.array([r for r in range(blk.row_count) if keep(b * rpb + r)], dtype=np.int32) for b, blk in enumerate(blocks)]
            assert res.selected_rows == sum(len(s) for s in sel)
            capped = batch.scan(flt, [0], max_selected_rows=max(res.selected_rows // 3, 1)) if res.selected_rows > 1 else None
            for gc in (2, 3, 4):
                for aggs in PATH_AGGS:
                    goff, out = res.group_by(gc, aggs)
                    for b, blk in enumerate(blocks):
                        cells = {c: truth[c][b * rpb:b * rpb + blk.row_count] for c in range(5, len(truth))}
                        want = exact_group_by_model(blk, gc, sel[b], aggs, cells)
                        assert np.array_equal(out[:, goff[b]:goff[b + 1]], want), (what, with_index, gc, b)
                    if capped is not None:    # the scan overflowed its capacity: the bitmap still selects every row
                        cgoff, cout = capped.group_by(gc, aggs)
                        assert np.array_equal(cgoff, goff) and np.array_equal(cout, out), (what, with_index, gc)
            if capped is not None:
                with pytest.raises(ob.ObGpuError) as e:
                    capped.info()
                assert e.value.code == ob.OB_BUF_NOT_ENOUGH
                capped.free()
            res.free()
    batch.close()


# ---- one table of more than 4 M rows: every CTA of the aggregate grid folds data ------------------------------------
@pytest.fixture(scope="module")
def big(ob):
    n = (1 << 22) + 12_345
    rng = np.random.default_rng(77)
    a = rng.integers(1 << 62, (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)    # INT near INT64_MAX: the low word
    a[rng.random(n) < 0.02] = np.iinfo(np.int64).min                                   # overflows in every CTA
    na = (rng.random(n) < 0.05).astype(np.uint8)
    u = rng.integers(1 << 63, M64 - 1, size=n, dtype=np.uint64, endpoint=True)         # UINT64 near 2^64 - 1
    u[rng.integers(0, n, size=50)] = 0
    w = np.where(rng.random(n) < 0.5, np.iinfo(np.int64).min, rng.integers(-(1 << 62), 1 << 62, size=n, dtype=np.int64))
    m = rng.integers(0, 100, size=n, dtype=np.int64)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, m), ob.Column(ob.OBJ_INT, ob.ENC_RAW, a, nulls=na),
            ob.Column(ob.OBJ_UINT64, ob.ENC_RAW, u.view(np.int64)), ob.Column(ob.OBJ_INT, ob.ENC_RAW, w)]
    table = ob.encode_table(cols, 2000)
    return table, m, np.where(na == 1, None, a.astype(object)), u.astype(object), w.astype(object)


def test_aggregates_over_four_million_rows(ob, ctx, big):
    table, m, a, u, w = big
    batch = ctx.open_batch(table)
    for flt, sel in ((None, np.ones(len(m), dtype=bool)), (ob.White(0, ob.WHITE_OP_LT, (50,)), m < 50)):
        res = batch.scan(flt, [0, 1, 2, 3])
        assert res.selected_rows == int(sel.sum())
        cols = {1: list(a[sel]), 2: list(u[sel]), 3: list(w[sel])}
        for c in (1, 2, 3):
            for kind in (COUNT, SUM, MIN, MAX):
                assert res.aggregate(kind, c) == fold(kind, cols[c]), (kind, c)
        for x, y in ((2, 3), (3, 3), (1, 2), (1, 3)):
            assert res.aggregate(SUM_PRODUCT, x, y) == fold(SUM_PRODUCT, cols[x], cols[y]), (x, y)
        res.free()
    batch.close()


# ---- the host pipeline folds per-batch aggregates -------------------------------------------------------------------
def test_pipeline_folds_batches_exactly(ob, ctx):
    from oceanbase_b200.pipeline import HostScanPipeline, batch_bounds
    rpb, bpb, n_blocks = 500, 8, 40
    n = rpb * n_blocks
    rng = np.random.default_rng(9)
    batch_of = np.arange(n) // rpb // bpb
    m = rng.integers(0, 99, size=n, dtype=np.int64)
    m[batch_of == 2] = 99                                            # batch 2 selects nothing
    s = rng.integers((1 << 63) - (1 << 58), (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)
    u = rng.integers(1 << 62, (1 << 63) + (1 << 62), size=n, dtype=np.uint64)
    u[batch_of == 0] |= np.uint64(1 << 63)                           # batch 0: every value above 2^63, the maximum too
    u[batch_of == 1] &= np.uint64((1 << 63) - 1)                     # batch 1: every value below 2^63, the minimum too
    u[np.nonzero(batch_of == 0)[0][17]] = np.uint64(M64 - 1)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(ob.OBJ_INT, ob.ENC_RAW, m),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, s), ob.Column(ob.OBJ_UINT64, ob.ENC_RAW, u.view(np.int64))]
    table = ob.encode_table(cols, rpb)
    flt = ob.White(1, ob.WHITE_OP_LT, (99,))
    aggs = [(COUNT, 2, -1), (SUM, 2, -1), (SUM, 3, -1), (MIN, 3, -1), (MAX, 3, -1), (MIN, 2, -1), (MAX, 2, -1), (SUM_PRODUCT, 3, 2)]
    sel = m < 99
    sv, uv = [int(x) for x in s[sel]], [int(x) for x in u[sel]]
    want = [fold(COUNT, sv), fold(SUM, sv), fold(SUM, uv), fold(MIN, uv), fold(MAX, uv), fold(MIN, sv), fold(MAX, sv),
            fold(SUM_PRODUCT, uv, sv)]
    # the inputs reach what the fold must survive: the extremes of u lie in different batches on either side of 2^63, and
    # the per-batch partial sums carry out of the low word when they are folded
    bounds = batch_bounds(n_blocks, bpb)
    parts = [[int(x) for x in s[b0 * rpb:b1 * rpb][sel[b0 * rpb:b1 * rpb]]] for b0, b1 in zip(bounds[:-1], bounds[1:])]
    assert not parts[2] and sum(sum(p) % M64 for p in parts) >= M64
    assert int(u[sel][batch_of[sel] == 0].max()) == want[4] >= 1 << 63 and int(u[sel][batch_of[sel] == 1].min()) == want[3] < 1 << 63
    pipe = HostScanPipeline(0, n_workers=3)
    try:
        out = pipe.scan(table, flt, [0, 1, 2, 3], blocks_per_batch=bpb, selectivity_hint=1.0, aggs=aggs, no_row_output=True)
    finally:
        pipe.close()
    assert out.selected_rows == int(sel.sum()) and len(out.batches) == len(bounds) - 1
    # the pipeline hands MIN / MAX back as the 64-bit image (int64), the scan result in the column's own order
    batch = ctx.open_batch(table)
    res = batch.scan(flt, [0, 1, 2, 3])
    for (kind, a, b), got, exp in zip(aggs, out.aggregates, want):
        single = res.aggregate(kind, a, b)
        assert single == exp, (kind, a)
        assert got == (to_i64(exp) if kind in (MIN, MAX) else exp), (kind, a)
    res.free()
    batch.close()
