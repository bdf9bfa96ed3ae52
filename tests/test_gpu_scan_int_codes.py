"""Batch integer codes (batch_codes.cuh): a range leaf (EQ / NE / LT / LE / GT / GE / BT) on a dictionary-coded fixed-width integer
column scanned with stage records is evaluated once per scan over the batch's distinct values, and the count kernel looks each row's
code up in that bitset; when every filter column is coded the count kernel's all-coded instantiation runs. Every scan here runs with
the codes on and with them off (OBGPU_STR_CODES=0: the per-block dictionary leaf) and is checked against a plain Python predicate
over the generated values.

Covered: every integer type the writer supports, signed and unsigned (the sign-fix types among them), byte-packed and bit-packed
refs, the type's minimum and maximum stored and as constants, constants between dictionary entries, NULL rows, AND and OR trees
mixing coded integer, coded string and uncoded columns, all-coded scans next to scans that are not, several batches scanned more
than once and closed and opened again, and a column above the 65 536-code cap (it keeps the per-block path). The writer stores
every PAX integer dictionary sorted, so the per-block path these scans are compared with is the sorted-interval one."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EQ, LE, LT, GE, GT, NE, BT, IN = range(8)   # OBGPU_WHITE_OP_*
RPB = 133
PLANS, RECORDS, CODED = 1, 2, 3              # OBGPU_COUNT_PIPE_*; 0: the small-block count kernel did not run

# (name, obj type, bits, signed)
TYPES = [("tinyint", 1, 8, True), ("smallint", 2, 16, True), ("mediumint", 3, 24, True), ("int32", 4, 32, True),
         ("int", 5, 64, True), ("utinyint", 6, 8, False), ("usmallint", 7, 16, False), ("umediumint", 8, 24, False),
         ("uint32", 9, 32, False), ("uint64", 10, 64, False), ("date", 19, 32, True), ("year", 21, 8, False)]


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
    monkeypatch.setenv("OBGPU_PIPE", "1")


def bounds(bits, signed):
    return (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if signed else (0, (1 << bits) - 1)


def as_i64(vals):
    """Python ints (unsigned up to 2^64 - 1) -> the int64 bit patterns the writer takes"""
    return np.array([v - (1 << 64) if v >= 1 << 63 else v for v in vals], dtype=np.int64)


def int_values(rng, n, bits, signed, n_distinct=40):
    """n values over a domain of spaced (even-offset) values with the type's minimum and maximum; about 1 in 9 NULL"""
    lo, hi = bounds(bits, signed)
    mid = [int(x) for x in rng.integers(0, 1 << min(bits - 2, 40), n_distinct - 2)]
    dom = sorted({lo, hi} | {lo + 2 * m + 2 for m in mid})
    vals = [dom[int(k)] for k in rng.integers(0, len(dom), n)]
    nulls = rng.random(n) < 0.11
    return vals, nulls, dom


def absent_between(dom):
    """a constant between two dictionary entries"""
    for a, b in zip(dom, dom[1:]):
        if b - a > 1:
            return a + 1
    raise AssertionError("no gap")


def leaf_pass(op, v, params):
    if v is None:
        return False
    c = params[0]
    if op == EQ: return v == c
    if op == NE: return v != c
    if op == LT: return v < c
    if op == LE: return v <= c
    if op == GT: return v > c
    if op == GE: return v >= c
    if op == BT: return params[0] <= v <= params[1]
    if op == IN: return v in params
    raise AssertionError(op)


def model(expr, cols, n):
    """selected row ids of the filter tree over the Python values (None: NULL)"""
    from oceanbase_b200 import And, Or

    def ev(e, i):
        if isinstance(e, And):
            return all(ev(c, i) for c in e.children)
        if isinstance(e, Or):
            return any(ev(c, i) for c in e.children)
        return leaf_pass(e.op, cols[e.col][i], e.params)
    return [i for i in range(n) if ev(expr, i)]


def count_kernel(ob, ctx):
    pcb, ctas, kern = C.c_int32(), C.c_int32(), C.c_int32()
    assert ob.capi.lib.obgpu_ctx_count_layout(ctx._h, C.byref(pcb), C.byref(ctas), C.byref(kern)) == 0
    return kern.value, ctas.value


def codes_state(ob, batch, col):
    state, n, ms = C.c_int32(), C.c_int32(), C.c_float()
    assert ob.capi.lib.obgpu_batch_string_codes(batch._h, col, C.byref(state), C.byref(n), C.byref(ms)) == 0
    return state.value, n.value


def scan_ids(batch, f):
    res = batch.scan(f, [0])
    try:
        return [int(x) for x in res.fetch_col(0)[0]] if res.selected_rows else []
    finally:
        res.free()


def check(ob, ctx, batch, monkeypatch, f, cols, n, on_kernel=None, name=""):
    """the scan with codes on and off against the model; on_kernel: the count instantiation(s) the scan may run with codes on"""
    want = model(f, cols, n)
    for knob in ("1", "0"):
        monkeypatch.setenv("OBGPU_STR_CODES", knob)
        got = scan_ids(batch, f)
        assert got == want, (name, knob, f, len(got), len(want), sorted(set(got) ^ set(want))[:10])
        if knob == "1" and on_kernel is not None:
            assert count_kernel(ob, ctx)[0] in np.atleast_1d(on_kernel), (name, f, count_kernel(ob, ctx))


def int_table(ob, rng, n, bits, signed, obj, byte_packing):
    vals, nulls, dom = int_values(rng, n, bits, signed)
    cols = [ob.Column(5, ob.ENC_RAW, np.arange(n, dtype=np.int64)),
            ob.Column(obj, ob.ENC_DICT, as_i64(vals), nulls=nulls.astype(np.uint8), byte_packing_only=byte_packing)]
    model_cols = {1: [None if z else v for v, z in zip(vals, nulls)]}
    return ob.encode_table(cols, RPB), model_cols, dom


@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
@pytest.mark.parametrize("tname,obj,bits,signed", TYPES, ids=[t[0] for t in TYPES])
def test_int_leaves_match_the_model(ob, ctx, monkeypatch, tname, obj, bits, signed, byte_packing):
    rng = np.random.default_rng(bits * 31 + obj * 7 + byte_packing)
    n = RPB * 30 + 7
    table, cols, dom = int_table(ob, rng, n, bits, signed, obj, byte_packing)
    lo, hi = bounds(bits, signed)
    consts = [lo, hi, dom[len(dom) // 2], absent_between(dom), lo + 1, hi - 1]
    batch = ctx.open_batch(table)
    try:
        for op in (EQ, NE, LT, LE, GT, GE):
            for c in consts:
                # a single leaf whose column is coded runs the all-coded count kernel (an empty range, e.g. LT min, is no record leaf)
                empty = (op == LT and c == lo) or (op == GT and c == hi)
                check(ob, ctx, batch, monkeypatch, ob.White(1, op, (c,)), cols, n, None if empty else CODED, (tname, op, c))
        for a, b in ((lo, hi), (dom[1], absent_between(dom)), (dom[2], dom[2]), (hi, lo)):
            check(ob, ctx, batch, monkeypatch, ob.White(1, BT, (a, b)), cols, n, None, (tname, "bt", a, b))
        state, n_codes = codes_state(ob, batch, 1)
        assert state == 1 and n_codes == len(set(v for v in cols[1] if v is not None)), (state, n_codes)
    finally:
        batch.close()


def mixed_table(ob, rng, n):
    """0 row id; 1 INT32 DICT (sign fix); 2 VARCHAR DICT; 3 UINT64 DICT; 4 INT RAW (no dictionary: plans); 5 SMALLINT DICT;
    6 UTINYINT DICT"""
    v1, z1, d1 = int_values(rng, n, 32, True)
    v3, z3, d3 = int_values(rng, n, 64, False)
    v5, z5, d5 = int_values(rng, n, 16, True, 12)
    v6, z6, d6 = int_values(rng, n, 8, False, 9)
    words = [b"", b"a", b"apple", b"apples and pears", b"banana", b"cherry-cherry-cherry"]
    s2 = [words[int(k)] for k in rng.integers(0, len(words), n)]
    z2 = rng.random(n) < 0.08
    v4 = [int(x) for x in rng.integers(-1000, 1000, n)]
    cols = [ob.Column(5, ob.ENC_RAW, np.arange(n, dtype=np.int64)),
            ob.Column(4, ob.ENC_DICT, as_i64(v1), nulls=z1.astype(np.uint8)),
            ob.Column(22, ob.ENC_DICT, s2, nulls=z2.astype(np.uint8)),
            ob.Column(10, ob.ENC_DICT, as_i64(v3), nulls=z3.astype(np.uint8), byte_packing_only=True),
            ob.Column(5, ob.ENC_RAW, np.array(v4, dtype=np.int64)),
            ob.Column(2, ob.ENC_DICT, as_i64(v5), nulls=z5.astype(np.uint8)),
            ob.Column(6, ob.ENC_DICT, as_i64(v6), nulls=z6.astype(np.uint8))]
    m = {1: [None if z else v for v, z in zip(v1, z1)], 2: [None if z else v for v, z in zip(s2, z2)],
         3: [None if z else v for v, z in zip(v3, z3)], 4: v4, 5: [None if z else v for v, z in zip(v5, z5)],
         6: [None if z else v for v, z in zip(v6, z6)]}
    return ob.encode_table(cols, RPB), m, (d1, d3, d5, d6)


def trees(ob, doms):
    And, Or, W = ob.And, ob.Or, ob.White
    d1, d3, d5, d6 = doms
    m1, m3 = d1[len(d1) // 2], d3[len(d3) // 3]
    return [   # (name, filter, count instantiation with codes on)
        ("and_int_int_str", And([W(1, GE, (m1,)), W(3, LT, (m3,)), W(2, IN, (b"apple", b"banana", b"nope"))]), CODED),
        ("and_str_first", And([W(2, NE, (b"cherry-cherry-cherry",)), W(1, LE, (d1[-2],)), W(3, GT, (d3[1],))]), CODED),
        ("or_int_str_int", Or([W(1, EQ, (m1,)), W(2, EQ, (b"",)), W(3, BT, (d3[2], d3[-3]))]), CODED),
        ("or_ne", Or([W(1, NE, (d1[0],)), W(3, EQ, (d3[-1],))]), CODED),
        ("and_same_col", And([W(1, GT, (d1[3],)), W(1, LT, (d1[-4],)), W(5, NE, (d5[1],))]), CODED),
        ("and_raw_col", And([W(1, LT, (m1,)), W(4, GT, (0,))]), (0, PLANS)),
        ("or_raw_col", Or([W(3, GE, (m3,)), W(4, EQ, (7,)), W(2, EQ, (b"a",))]), (0, PLANS)),
        ("and_five_cols", And([W(1, GE, (d1[1],)), W(3, NE, (m3,)), W(2, NE, (b"banana",)), W(5, LE, (d5[-2],)), W(6, GT, (d6[1],))]),
         RECORDS),
        ("or_five_cols", Or([W(6, EQ, (d6[2],)), W(5, EQ, (d5[3],)), W(3, EQ, (m3,)), W(1, EQ, (m1,)), W(2, EQ, (b"cherry-cherry-cherry",))]),
         RECORDS),
    ]


def test_trees_mix_coded_and_uncoded_columns(ob, ctx, monkeypatch):
    rng = np.random.default_rng(2024)
    n = RPB * 40 + 17
    table, cols, doms = mixed_table(ob, rng, n)
    batch = ctx.open_batch(table)
    try:
        for name, f, kern in trees(ob, doms):
            check(ob, ctx, batch, monkeypatch, f, cols, n, kern, name)
        for c in (1, 2, 3, 5):
            assert codes_state(ob, batch, c)[0] == 1, c
        assert codes_state(ob, batch, 4)[0] == 0   # its leaves never take records: nothing was built
        # the all-coded count kernel fits more CTAs per SM than the record kernel
        monkeypatch.setenv("OBGPU_STR_CODES", "1")
        scan_ids(batch, trees(ob, doms)[0][1])
        assert count_kernel(ob, ctx)[1] >= 10, count_kernel(ob, ctx)
    finally:
        batch.close()


def test_several_batches_rescanned_and_reopened(ob, ctx, monkeypatch):
    rng = np.random.default_rng(77)
    made = [mixed_table(ob, rng, RPB * 20 + 5), mixed_table(ob, rng, RPB * 13 + 100)]
    for _ in range(2):   # open, scan twice, close; then again
        batches = [ctx.open_batch(t) for t, _, _ in made]
        try:
            for _ in range(2):
                for (t, cols, doms), batch in zip(made, batches):
                    for name, f, kern in trees(ob, doms)[::2]:
                        check(ob, ctx, batch, monkeypatch, f, cols, t.total_rows, kern, name)
            for batch in batches:
                assert all(codes_state(ob, batch, c)[0] == 1 for c in (1, 2, 3))
        finally:
            for batch in batches:
                batch.close()


def test_column_over_the_code_cap_keeps_the_per_block_path(ob, ctx, monkeypatch):
    n = 70_000
    vals = np.arange(n, dtype=np.int64) * 3 - 50_000   # all distinct: a DICT of 133 entries in every block
    cols = [ob.Column(5, ob.ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(5, ob.ENC_DICT, vals)]
    batch = ctx.open_batch(ob.encode_table(cols, RPB))
    try:
        m = {1: [int(v) for v in vals]}
        for f in (ob.White(1, EQ, (int(vals[69_999]),)), ob.White(1, LT, (-49_990,)), ob.White(1, NE, (int(vals[0]),)),
                  ob.White(1, BT, (1, 301))):
            check(ob, ctx, batch, monkeypatch, f, m, n, RECORDS)
        assert codes_state(ob, batch, 1)[0] == -2   # OBGPU_CODES_OVER_CAP
    finally:
        batch.close()
