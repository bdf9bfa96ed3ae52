"""Batch codes (batch_codes.cuh) on the device against the plain value model of tests/test_scan_codes_model.py, whose CPU half
proves the tables hold what each case below relies on.

Every scan runs with the codes on and off (OBGPU_STR_CODES) on the pipelined kernels (OBGPU_PIPE=1), and on the general kernels
(OBGPU_PIPE=0, which never read codes), and must equal the model in: selected_rows, fetch_row_ids, fetch_sel_offsets, every
projected column -- the filter columns included -- at its element width with its NULL bits, and (codes on) one aggregate fold. With
the codes on it also checks which count instantiation ran and each filter column's code state; where a column is coded, n_codes
is the model's distinct count: within one batch a value has exactly one code.

Cases: 1. every integer type with blocks of different dictionary layouts, -1 / 0 / 1 / the extremes and their neighbours, byte-
and bit-packed refs, every range op around each of them; 2. CS INT_DICT / STR_DICT under three stream codecs, a PAX twin, one batch
of PAX and CS blocks, CS columns with an all-NULL block and with const-encoded refs (these, CS string dictionaries and the mixed
encodings of case 4 have no stage record that serves the filter: no scan builds their codes, state 0, and they keep the region
path); 3. thousands of strings of one length whose
hash tags collide, pairs among them sharing the home slot, the empty string, bytes >= 0x80 and NUL; 4. OBGPU_ENC_AUTO columns mixing
DICT with RAW / RLE / CONST blocks; 5. 65 536 and 65 537 distinct values; 6. the skip index settling blocks TRUE and FALSE and
leaves constant inside uncertain blocks, on the coded and the record instantiation; 7. every way a batch is opened, each scanned
twice (cached codes), closed and reopened; 8. the bench's cfg3 segment at its own block cut, against a numpy rebuild of its seeds."""
import ctypes as C

import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM, fold
from test_scan_codes_model import (BT, CAP, CS_MODES, EQ, GE, GT, IN, LE, LT, M64, NE, RPB, TYPE_IDS, auto_table, bench_model,
                                   bench_string, bench_workload, cap_table, collision_pool, concat_table, cs_table,
                                   cs_uncodable_table, int_filters, int_layout_table, open_table, string_table)
from test_gpu_scan_int_codes import TYPES, bounds

pytestmark = pytest.mark.gpu

PLANS, RECORDS, CODED = 1, 2, 3                    # OBGPU_COUNT_PIPE_*; 0: the small-block count kernel did not run
OVER_CAP = -2                                      # OBGPU_CODES_OVER_CAP


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def pipe(monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", "1")      # batches are opened with stage records


def count_kernel(ob, ctx):
    pcb, ctas, kern = C.c_int32(), C.c_int32(), C.c_int32()
    assert ob.capi.lib.obgpu_ctx_count_layout(ctx._h, C.byref(pcb), C.byref(ctas), C.byref(kern)) == 0
    return kern.value


def codes_state(ob, batch, col):
    state, n, ms = C.c_int32(), C.c_int32(), C.c_float()
    assert ob.capi.lib.obgpu_batch_string_codes(batch._h, col, C.byref(state), C.byref(n), C.byref(ms)) == 0
    return state.value, n.value


def starts(t, image=None):
    """first row of every block, then the total (from the block headers)"""
    img = t.image if image is None else image
    rows = [int(img.image[int(o) + 16:int(o) + 20].view(np.uint32)[0]) for o in img.offsets]
    return np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)


def check_result(res, t, want, proj, start, what):
    assert res.selected_rows == len(want), (what, res.selected_rows, len(want))
    w = np.asarray(want, dtype=np.int64)
    assert np.array_equal(res.fetch_sel_offsets(), np.searchsorted(w, start)), what
    if not want:
        return
    blk = np.searchsorted(start, w, side="right") - 1
    assert np.array_equal(res.fetch_row_ids(), (w - start[blk]).astype(np.int32)), what
    for i, c in enumerate(proj):
        data, _, nulls = res.fetch_col(i)
        null = np.unpackbits(np.ascontiguousarray(nulls).view(np.uint8), bitorder="little")[:len(want)].astype(bool)
        cells = [t.cells[c][r] for r in want]
        assert null.tolist() == [v is None for v in cells], (what, c)
        if t.widths[c]:
            mask = (1 << 8 * t.widths[c]) - 1
            assert data.itemsize == t.widths[c], (what, c)
            got = [int(x) for x, z in zip(data.tolist(), null) if not z]
            assert got == [v & mask for v in cells if v is not None], (what, c)
        else:
            heap, off = res.fetch_strings(i)
            assert [None if z else bytes(heap[off[j]:off[j + 1]]) for j, z in enumerate(null)] == cells, (what, c)


def check_aggs(res, t, want, proj, what):
    """SUM / MIN / MAX / COUNT of the first projected non-key integer column against the exact fold"""
    i = next((i for i, c in enumerate(proj) if c != 0 and t.widths[c]), None)
    if i is None:
        return
    cells = [t.cells[proj[i]][r] for r in want]
    for kind in (COUNT, SUM, MIN, MAX):
        assert res.aggregate(kind, i) == fold(kind, cells), (what, kind)


def check(ob, ctx, batch, t, monkeypatch, flt, kernel=None, start=None, proj=None, pipe0=True, aggs=True, name=""):
    """the scan with codes on and off on the pipelined kernels and once on the general ones, against the model; kernel: the count
    instantiation(s) the scan must run with codes on"""
    proj = t.proj if proj is None else proj
    start = starts(t) if start is None else start
    want = t.selected(flt)
    runs = [("1", "1"), ("1", "0")] + ([("0", "1")] if pipe0 else [])
    for pipe, knob in runs:
        monkeypatch.setenv("OBGPU_PIPE", pipe)
        monkeypatch.setenv("OBGPU_STR_CODES", knob)
        res = batch.scan(flt, proj, want_row_ids=True)
        try:
            what = (t.name, name, pipe, knob, flt)
            check_result(res, t, want, proj, start, what)
            if pipe == "1" and knob == "1":
                if kernel is not None:
                    assert count_kernel(ob, ctx) in np.atleast_1d(kernel), (what, count_kernel(ob, ctx))
                if aggs:
                    check_aggs(res, t, want, proj, what)
        finally:
            res.free()
    monkeypatch.setenv("OBGPU_PIPE", "1")
    monkeypatch.setenv("OBGPU_STR_CODES", "1")


def assert_states(ob, batch, t, states):
    """col -> expected state; a coded column has one code per distinct non-NULL value of the model"""
    for col, want in states.items():
        state, n = codes_state(ob, batch, col)
        assert state == want, (t.name, col, state, n)
        if state == 1:
            assert n == t.distinct(col), (t.name, col, n, t.distinct(col))


# ---- 1. integer layouts ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
@pytest.mark.parametrize("tname", TYPE_IDS)
def test_integer_layouts(ob, ctx, monkeypatch, tname, byte_packing):
    t = int_layout_table(tname, byte_packing)
    _, _, bits, signed = next(x for x in TYPES if x[0] == tname)
    lo, hi = bounds(bits, signed)
    batch = ctx.open_batch(t.image)
    try:
        start = starts(t)
        for j, f in enumerate(int_filters(ob, tname)):
            empty = (f.op == LT and f.params[0] == lo) or (f.op == GT and f.params[0] == hi)
            kern = None if empty or f.op == BT else CODED
            check(ob, ctx, batch, t, monkeypatch, f, kern, start, pipe0=j % 3 == 0, aggs=j % 4 == 0, name=j)
        assert_states(ob, batch, t, {1: 1})
    finally:
        batch.close()


# ---- 2. CS dictionaries ----------------------------------------------------------------------------------------------------
def cs_filters(ob):
    W, And, Or = ob.White, ob.And, ob.Or
    return [W(1, EQ, (-1,)), W(1, LE, (0,)), W(1, GT, (1,)), W(1, BT, (-1000, -1)), W(2, EQ, (-1,)), W(2, LT, (-1,)),
            W(2, GE, (-(1 << 15),)), W(3, EQ, (M64,)), W(3, GE, (1 << 63,)), W(3, LT, ((1 << 63) - 1,)), W(4, EQ, (b"\x80",)),
            W(4, IN, (b"", b"a\x00", b"zz" * 7)), W(4, NE, (b"a",)),
            And([W(1, NE, (0,)), W(2, GE, (-1,)), W(4, NE, (b"apple",))]), Or([W(3, EQ, (M64,)), W(1, EQ, (-1000,)), W(4, EQ, (b"",))])]


@pytest.mark.parametrize("which", ["pax"] + ["cs%d" % m for m in CS_MODES] + ["pax+cs"])
def test_cs_dictionaries(ob, ctx, monkeypatch, which):
    t = {"pax": lambda: cs_table(1, pax=True), "pax+cs": concat_table}.get(which, lambda: cs_table(int(which[2:])))()
    batch = ctx.open_batch(t.image)
    try:
        start = starts(t)
        for j, f in enumerate(cs_filters(ob)):
            check(ob, ctx, batch, t, monkeypatch, f, CODED if which == "pax" else None, start, name=j)
        # a CS string dictionary keeps its bytes in the block's all-string-data area: no stage record serves the filter, so its
        # codes are never built (state 0) and a leaf on it keeps the region path
        assert_states(ob, batch, t, {1: 1, 2: 1, 3: 1, 4: 1 if which == "pax" else 0})
    finally:
        batch.close()


def test_cs_columns_that_cannot_be_coded(ob, ctx, monkeypatch):
    t = cs_uncodable_table()
    W, And, Or = ob.White, ob.And, ob.Or
    batch = ctx.open_batch(t.image)
    try:
        for j, f in enumerate([W(1, EQ, (-1,)), W(1, GE, (0,)), W(2, EQ, (42,)), W(2, LT, (-3,)), W(3, LE, (5,)),
                               And([W(3, GE, (0,)), W(1, NE, (2,))]), Or([W(2, NE, (42,)), W(3, EQ, (-3,))])]):
            check(ob, ctx, batch, t, monkeypatch, f, (0, PLANS) if j != 4 else CODED, name=j)
        # an all-NULL block (a CONST plan) or const-encoded refs: the column's stage records do not serve the filter, so no scan
        # takes records on it and its codes are never built; column 3 alone codes
        assert_states(ob, batch, t, {1: 0, 2: 0, 3: 1})
    finally:
        batch.close()


# ---- 3. strings -------------------------------------------------------------------------------------------------------------
def test_strings_with_colliding_tags(ob, ctx, monkeypatch):
    t = string_table()
    pool, n_pairs = collision_pool()
    W, And, Or = ob.White, ob.And, ob.Or
    pairs = pool[:2 * n_pairs]
    fs = [(W(1, EQ, (s,)), CODED) for s in pairs[:16]]
    fs += [(W(1, NE, (pairs[0],)), CODED), (W(1, IN, tuple(pairs[1:12:2]) + (b"\x80c999999999\xff",)), CODED),
           (W(1, IN, (pairs[2], pairs[3], b"", b"\x00" * 12)), CODED),
           (W(2, EQ, (b"",)), CODED), (W(2, EQ, (b"a\x80b",)), CODED), (W(2, EQ, (b"a\xffb",)), CODED), (W(2, NE, (b"\x00",)), CODED),
           (W(2, IN, (b"a\x00b", b"\x00" * 12, b"\xff" * 12)), CODED),
           (And([W(1, NE, (pairs[4],)), W(2, EQ, (b"a\x7fb",)), W(4, GE, (0,))]), CODED),
           (Or([W(1, EQ, (pairs[5],)), W(2, EQ, (b"",)), W(4, EQ, (-3,))]), CODED),
           (And([W(3, GT, (0,)), W(1, EQ, (pairs[6],))]), None), (Or([W(1, EQ, (pairs[7],)), W(3, EQ, (7,))]), None)]
    batch = ctx.open_batch(t.image)
    try:
        start = starts(t)
        for j, (f, kern) in enumerate(fs):
            check(ob, ctx, batch, t, monkeypatch, f, kern, start, pipe0=j % 2 == 0, name=j)
        assert_states(ob, batch, t, {1: 1, 2: 1, 4: 1})
    finally:
        batch.close()


# ---- 4. mixed encodings -----------------------------------------------------------------------------------------------------
def test_auto_columns_mixing_encodings_keep_the_region_path(ob, ctx, monkeypatch):
    t = auto_table()
    W, And, Or = ob.White, ob.And, ob.Or
    batch = ctx.open_batch(t.image)
    try:
        for j, f in enumerate([W(1, EQ, (-1,)), W(1, GT, (0,)), W(1, BT, (-9, 9)), W(2, EQ, (b"s1",)), W(2, NE, (b"s999",)),
                               And([W(3, LT, (10,)), W(1, NE, (-1,))]), Or([W(2, EQ, (b"s0",)), W(3, EQ, (4,))])]):
            check(ob, ctx, batch, t, monkeypatch, f, (0, PLANS), name=j)
        # RAW / RLE / CONST blocks have no dictionary record: no scan takes records on the column, its codes are never built
        assert_states(ob, batch, t, {1: 0, 2: 0})
    finally:
        batch.close()


# ---- 5. the code cap --------------------------------------------------------------------------------------------------------
def test_cap_boundary(ob, ctx, monkeypatch):
    t = cap_table()
    W = ob.White
    v1 = sorted(set(t.cells[1]))
    v2 = sorted(set(t.cells[2]))
    batch = ctx.open_batch(t.image)
    try:
        start = starts(t)
        for j, f in enumerate([W(1, EQ, (v1[-1],)), W(1, EQ, (v1[0],)), W(1, EQ, (v1[CAP // 2],)), W(1, NE, (v1[7],)),
                               W(1, GE, (v1[-3],)), W(1, BT, (v1[100], v1[160])), W(1, LT, (v1[0] + 1,))]):
            check(ob, ctx, batch, t, monkeypatch, f, CODED, start, pipe0=j < 2, name=j)
        assert_states(ob, batch, t, {1: 1})
        assert codes_state(ob, batch, 1)[1] == CAP
        for j, f in enumerate([W(2, EQ, (v2[-1],)), W(2, NE, (v2[0],)), W(2, LE, (v2[2],))]):
            check(ob, ctx, batch, t, monkeypatch, f, RECORDS, start, pipe0=False, name=("over", j))
        assert_states(ob, batch, t, {2: OVER_CAP})
    finally:
        batch.close()


# ---- 6. skip index ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tname", ["int", "smallint", "uint64", "int32"])
def test_skip_index_settled_blocks(ob, ctx, monkeypatch, tname):
    t = int_layout_table(tname, False)
    _, _, bits, signed = next(x for x in TYPES if x[0] == tname)
    lo, hi = bounds(bits, signed)
    W, And, Or = ob.White, ob.And, ob.Or
    rows, offs = ob.table_agg_rows(t.cols, [1], RPB)
    batch = ctx.open_batch(t.image)
    batch.set_agg_rows(rows, offs)
    # GT 7: the small-value blocks settle FALSE; GE lo: NULL-free blocks settle TRUE; LE hi inside an uncertain block is a constant
    # leaf next to an uncertain NE
    fs = [W(1, GT, (7,)), W(1, GE, (lo,)), W(1, LE, (7,)), And([W(1, LE, (hi,)), W(1, NE, (3,))]), And([W(1, GE, (0,)), W(1, LE, (7,))]),
          Or([W(1, EQ, (5,)), W(1, GT, (7,))]), Or([W(1, LT, (1,)), W(1, GE, (lo,))])]
    settled = [0, 0]
    try:
        start = starts(t)
        for j, f in enumerate(fs):
            check(ob, ctx, batch, t, monkeypatch, f, CODED, start, name=j)
            for knob, kern in (("1", CODED), ("0", RECORDS)):
                monkeypatch.setenv("OBGPU_STR_CODES", knob)
                res = batch.scan(f, [0, 1], want_row_ids=True)
                try:
                    check_result(res, t, t.selected(f), [0, 1], start, (tname, j, knob))
                    assert count_kernel(ob, ctx) == kern, (j, knob, count_kernel(ob, ctx))
                    fa, tr = res.skip_info()
                    settled[0] += fa
                    settled[1] += tr
                finally:
                    res.free()
        assert settled[0] > 0 and settled[1] > 0, settled
        assert_states(ob, batch, t, {1: 1})
    finally:
        batch.close()


# ---- 7. open paths ----------------------------------------------------------------------------------------------------------
def open_filters(ob, k):
    W, And, Or = ob.White, ob.And, ob.Or
    return [[And([W(1, GE, (-1,)), W(2, EQ, (b"a\x80b",))]), Or([W(1, EQ, (-1,)), W(3, GT, (1 << 63,))]), W(1, LE, (2,))],
            [And([W(1, LT, (1,)), W(2, NE, (b"",))]), Or([W(1, EQ, ((1 << 63) - 1,)), W(3, EQ, (M64,))]), W(3, BT, (1, (1 << 63) - 1))]][k]


@pytest.mark.parametrize("path", ["host", "device", "device_no_host_view", "lz4", "zstd", "macro"])
def test_open_paths(ob, ctx, monkeypatch, path):
    import torch
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    t = open_table()
    keep = None

    def opened():
        nonlocal keep
        if path == "host":
            return ctx.open_batch(t.image)
        if path in ("device", "device_no_host_view"):
            keep = torch.from_numpy(t.image.image).cuda()
            return ctx.open_batch(t.image, device_image_ptr=keep.data_ptr(), host_view=path == "device", image_size=t.image.image.size)
        if path in ("lz4", "zstd"):
            comp = ob.capi.COMPRESSOR_LZ4 if path == "lz4" else ob.capi.COMPRESSOR_ZSTD_1_3_8
            return ctx.open_batch(compress_table(t.image, comp), compressor=comp)
        mi = build_macro_blocks(t.image, t.obj_types, 1, macro_block_size=64 << 10)
        return ob.PageBatch.from_macro_blocks(ctx, mi.image, 64 << 10, mi.n_macro)

    start = starts(t)
    for _ in range(2):   # open, scan with two sets of constants (the second finds the codes built), close; then again
        batch = opened()
        try:
            assert batch.n_blocks == t.image.n_blocks and batch.total_rows == t.n
            for k in (0, 1):
                for j, f in enumerate(open_filters(ob, k)):
                    check(ob, ctx, batch, t, monkeypatch, f, CODED, start, pipe0=k == 0, name=(path, k, j))
            assert_states(ob, batch, t, {1: 1, 2: 1, 3: 1})
        finally:
            batch.close()
            keep = None


# ---- 8. the bench shape -----------------------------------------------------------------------------------------------------
def test_bench_segment(ob, ctx, monkeypatch):
    w = bench_workload()
    ints, strs = bench_model()
    n = w.table.total_rows
    W, And = ob.White, ob.And
    c0 = ints[0][0][ints[0][1]]
    c3 = ints[3][0][ints[3][1]]
    r9 = strs[9][1]
    base = w.filter.children
    in_list = base[2].params
    ranks_in = [k for k in range(1024) if bench_string(strs, 9, k) in set(in_list)]
    variants = [(w.filter, (c0 == base[0].params[0]) & (c3 < 2_000_000) & np.isin(r9, ranks_in))]
    k1 = int(ints[0][0][3])
    variants.append((And([W(0, EQ, (k1,)), W(3, LT, (500_000,)), W(9, IN, in_list)]), (c0 == k1) & (c3 < 500_000) & np.isin(r9, ranks_in)))
    one = [k for k in range(1024) if bench_string(strs, 9, k) == bench_string(strs, 9, 7)]
    variants.append((And([W(0, NE, (base[0].params[0],)), W(3, GE, (4_000_000,)), W(9, IN, (bench_string(strs, 9, 7),))]),
                     (c0 != base[0].params[0]) & (c3 >= 4_000_000) & np.isin(r9, one)))
    start = starts(None, w.table)
    batch = ctx.open_batch(w.table)
    try:
        for j, (f, mask) in enumerate(variants):
            want = np.flatnonzero(mask)
            for knob in ("1", "0"):
                monkeypatch.setenv("OBGPU_STR_CODES", knob)
                res = batch.scan(f, w.proj, want_row_ids=True)
                try:
                    assert res.selected_rows == len(want), (j, knob)
                    if knob == "1":
                        assert count_kernel(ob, ctx) == CODED
                    assert np.array_equal(res.fetch_sel_offsets(), np.searchsorted(want, start)), (j, knob)
                    blk = np.searchsorted(start, want, side="right") - 1
                    assert np.array_equal(res.fetch_row_ids(), (want - start[blk]).astype(np.int32)), (j, knob)
                    for i, c in enumerate(w.proj):
                        data, _, nulls = res.fetch_col(i)
                        assert not np.unpackbits(np.ascontiguousarray(nulls).view(np.uint8))[:len(want)].any()
                        if c < 8:
                            vals, ranks = ints[c]
                            assert np.array_equal(data.view(np.int64), vals[ranks[want]]), (j, knob, c)
                        else:
                            heap, off = res.fetch_strings(i)
                            ranks = strs[c][1]
                            assert [bytes(heap[off[q]:off[q + 1]]) for q in range(len(want))] == \
                                [bench_string(strs, c, int(k)) for k in ranks[want]], (j, knob, c)
                    if knob == "1":
                        vals, ranks = ints[w.proj[0]]
                        sel = [int(x) for x in vals[ranks[want]]]
                        for kind in (COUNT, SUM, MIN, MAX):
                            assert res.aggregate(kind, 0) == fold(kind, sel), (j, kind)
                finally:
                    res.free()
        for c in (0, 3, 9):
            state, nc = codes_state(ob, batch, c)
            assert state == 1, (c, state)
        assert codes_state(ob, batch, 0)[1] == len(set(c0.tolist()))
        assert codes_state(ob, batch, 3)[1] == len(set(c3.tolist()))
        assert codes_state(ob, batch, 9)[1] == len({bench_string(strs, 9, int(k)) for k in np.unique(r9)})
    finally:
        batch.close()
