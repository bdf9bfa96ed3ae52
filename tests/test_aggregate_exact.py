"""Exact integer folds for the pushed-down aggregates (COUNT / SUM / SUM_PRODUCT / MIN / MAX, obgpu_result_aggregate) and
pushdown GROUP BY (obgpu_block_group_by / obgpu_result_group_by), over every integer class, type extreme and value codec.

CPU half: the tables tests/test_gpu_aggregate_exact.py scans are what they claim to be -- the oracle decodes every cell back
to the generated value (type extremes included), the writer really chose the intended codec, and the Python reference fold
agrees with a brute-force fold over the oracle's cells done in 64-bit words with explicit carries.

Reference semantics (include/obgpu_scan.h, obgpu_result_aggregate): signed classes are sign-extended, unsigned ones (YEAR
included) zero-extended; SUM and SUM_PRODUCT are exact, then reduced to signed 128-bit two's complement; MIN / MAX use the
column's own order; NULL cells are skipped, and a SUM_PRODUCT row is skipped when either side is NULL."""
import functools

import numpy as np
import pytest

import oracle_binding as ora

M64, M128 = 1 << 64, 1 << 128
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
COUNT, SUM, SUM_PRODUCT, MIN, MAX = range(5)            # OBGPU_AGG_*
ENC_RAW, ENC_DICT, ENC_RLE, ENC_CONST, ENC_IBD = range(5)
ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STR_DICT = 16, 17, 19
OBJ_INT, OBJ_VARCHAR = 5, 22

# name -> (ObObjType, minimum, maximum); datum length 1 for YEAR, 4 for DATE, 8 for the rest
TYPES = {
    "tinyint": (1, -(1 << 7), (1 << 7) - 1),
    "smallint": (2, -(1 << 15), (1 << 15) - 1),
    "mediumint": (3, -(1 << 23), (1 << 23) - 1),
    "int32": (4, -(1 << 31), (1 << 31) - 1),
    "int": (5, I64_MIN, I64_MAX),
    "utinyint": (6, 0, (1 << 8) - 1),
    "usmallint": (7, 0, (1 << 16) - 1),
    "umediumint": (8, 0, (1 << 24) - 1),
    "uint32": (9, 0, (1 << 32) - 1),
    "uint64": (10, 0, M64 - 1),
    "date": (19, -(1 << 31), (1 << 31) - 1),
    "year": (21, 0, 255),
}
# name -> (encoding, byte_packing_only, value shape); PAX codecs below 16, CS codecs from 16 on
CODECS = {
    "raw": (ENC_RAW, False, "free"),
    "raw_bp": (ENC_RAW, True, "free"),
    "dict": (ENC_DICT, False, "pool"),
    "rle": (ENC_RLE, False, "runs"),
    "const": (ENC_CONST, False, "const"),
    "const_exc": (ENC_CONST, False, "const_exc"),
    "ibd": (ENC_IBD, False, "free"),
    "cs_integer": (ENC_CS_INTEGER, False, "free"),
    "cs_int_dict": (ENC_CS_INT_DICT, False, "pool"),
}
# the ObColumnHeader::type_ (PAX) / ObCSColumnHeader::type_ (CS) each codec must leave in every block
HEADER_TYPE = {ENC_RAW: 0, ENC_DICT: 1, ENC_RLE: 2, ENC_CONST: 3, ENC_IBD: 4, ENC_CS_INTEGER: 0, ENC_CS_INT_DICT: 2, ENC_CS_STR_DICT: 3}

N_ROWS, RPB = 1500, 250
# store columns of a matrix table
K, M, W, VA, VB, VN = range(6)       # row number, 0..99, INT with INT extremes (10 % NULL), value columns: 0 % / 10 % / 100 % NULL
GROUP_COLS_PAX = {"dict_int": 6, "dict_str": 7, "rle": 8, "const": 9}
GROUP_COLS_CS = {"cs_int_dict": 6, "cs_str_dict": 7}
# rows of group key 3 hold the type's maximum in VA, rows of key 5 its minimum (MIN / MAX == the fold's initial key for
# INT and UINT64); rows of key 7 are NULL in VB (a group whose only rows are NULL in the value column)
KEY_MAX, KEY_MIN, KEY_VB_NULL = 3, 5, 7


def vn_encoding(enc):
    """the codec of the all-NULL column: the writer's DICT and RLE refuse a column without a value, and INTEGER_BASE_DIFF has
    no base to take; such a column is CONST of NULL (DICT, RLE) or RAW there"""
    return {ENC_DICT: ENC_CONST, ENC_RLE: ENC_CONST, ENC_IBD: ENC_RAW}.get(enc, enc)


def is_cs(codec):
    return CODECS[codec][0] >= 16


def datum_len(obj_type):
    return 1 if obj_type == 21 else (4 if obj_type == 19 else 8)


def specials(tname):
    _, lo, hi = TYPES[tname]
    out = [lo, hi, 0] + ([-1] if lo < 0 else [])
    if tname == "uint64":
        out += [1 << 63, (1 << 63) - 1]
    return out


def to_i64(v):
    """the 64-bit image of v as a signed int64 (what int64 outputs of the C-ABI carry)"""
    v &= M64 - 1
    return v - M64 if v >= 1 << 63 else v


def wrap128(v):
    v %= M128
    return v - M128 if v >= 1 << 127 else v


def _draw(rng, lo, hi, size):
    return [lo + int(x) for x in rng.integers(0, hi - lo + 1, size=size, dtype=np.uint64).tolist()] if hi - lo >= 1 << 63 else \
        [int(x) for x in rng.integers(lo, hi + 1, size=size, dtype=np.int64).tolist()]


def gen_values(rng, tname, shape, n, bias):
    """n values of the type: type extremes mixed with draws from the upper (bias 'hi') or lower ('lo') half of its range,
    shaped for the codec (free values / a small pool / runs of pool values / one dominant value)"""
    _, lo, hi = TYPES[tname]
    mid = lo + (hi - lo) // 2
    sp = specials(tname)
    rlo, rhi = (mid, hi) if bias == "hi" else (lo, mid)
    if shape == "free":
        v = _draw(rng, rlo, rhi, n)
        pick = rng.random(n) < 0.35
        idx = rng.integers(0, len(sp), size=n)
        return [sp[i] if p else x for x, p, i in zip(v, pick.tolist(), idx.tolist())]
    pool = sp + _draw(rng, rlo, rhi, 6)
    if shape == "pool":
        return [pool[i] for i in rng.integers(0, len(pool), size=n).tolist()]
    if shape == "runs":
        out = []
        while len(out) < n:
            out += [pool[int(rng.integers(0, len(pool)))]] * int(rng.integers(1, 13))
        return out[:n]
    dominant = hi if bias == "hi" else lo
    out = [dominant] * n
    if shape == "const_exc":            # one exception every 37 rows: at most 7 per 250-row block (the writer takes <= 10 %)
        for i in range(11, n, 37):
            out[i] = pool[i % len(pool)]
    return out


def null_mask(rng, shape, n, rate):
    if rate >= 1.0:
        return np.ones(n, dtype=np.uint8)
    if shape in ("const", "const_exc"):
        # NULL is an exception of a CONST column too: a fixed stride keeps every block under the writer's exception limit
        m = np.zeros(n, dtype=np.uint8)
        m[7::25] = 1
        return m
    return (rng.random(n) < rate).astype(np.uint8)


def as_store(values):
    """Python ints -> the int64 array the writer takes (unsigned 64-bit values as their two's-complement image)"""
    return np.array([to_i64(v) for v in values], dtype=np.int64)


class Spec:
    """One generated table: the writer's columns plus the true value (Python int or None) of every cell"""

    def __init__(self, cols, truth, rpb, group_cols, obj_types, shape):
        self.cols, self.truth, self.rpb, self.group_cols, self.obj_types, self.shape = cols, truth, rpb, group_cols, obj_types, shape
        self.n = len(truth[0])


def with_nulls(values, mask):
    return [None if m else v for v, m in zip(values, mask.tolist())] if mask is not None else list(values)


@functools.lru_cache(maxsize=None)
def matrix_spec(tname, codec, n=N_ROWS, rpb=RPB, seed=0):
    import oceanbase_b200 as ob
    obj, lo, hi = TYPES[tname]
    enc, bp, shape = CODECS[codec]
    rng = np.random.default_rng(1000 * list(TYPES).index(tname) + 10 * list(CODECS).index(codec) + seed)
    base = ENC_CS_INTEGER if is_cs(codec) else ENC_RAW
    gkey = rng.integers(0, 12, size=n)
    va = gen_values(rng, tname, shape, n, "hi")
    vb = gen_values(rng, tname, shape, n, "lo")
    if shape in ("free", "pool"):     # group ties (see KEY_MAX); RLE / CONST shapes keep their structure
        va = [hi if g == KEY_MAX else (lo if g == KEY_MIN else x) for x, g in zip(va, gkey.tolist())]
    nb = null_mask(rng, shape, n, 0.10)
    if shape not in ("const", "const_exc"):
        nb[gkey == KEY_VB_NULL] = 1
    w = gen_values(rng, "int", "free", n, "lo")
    nw = (rng.random(n) < 0.10).astype(np.uint8)
    k = list(range(n))
    m = [int(x) for x in rng.integers(0, 100, size=n).tolist()]
    vn = gen_values(rng, tname, shape, n, "hi")
    nn = np.ones(n, dtype=np.uint8)
    cols = [ob.Column(OBJ_INT, base, as_store(k)), ob.Column(OBJ_INT, base, as_store(m)), ob.Column(OBJ_INT, base, as_store(w), nulls=nw)]
    cols += [ob.Column(obj, enc, as_store(v), nulls=nl, byte_packing_only=bp) for v, nl in ((va, None), (vb, nb))]
    cols.append(ob.Column(obj, vn_encoding(enc), as_store(vn), nulls=nn, byte_packing_only=bp))
    truth = [k, m, with_nulls(w, nw), va, with_nulls(vb, nb), with_nulls(vn, nn)]
    types = [OBJ_INT, OBJ_INT, OBJ_INT, obj, obj, obj]
    words = [b"g%02d" % i + b"#" * (i % 5) for i in range(12)]
    ng = (rng.random(n) < 0.05).astype(np.uint8)
    gint = [int(g) * 1000 - 5000 for g in gkey.tolist()]
    gstr = [words[g] for g in gkey.tolist()]
    if is_cs(codec):
        group_cols = dict(GROUP_COLS_CS)
        cols += [ob.Column(OBJ_INT, ENC_CS_INT_DICT, as_store(gint), nulls=ng), ob.Column(OBJ_VARCHAR, ENC_CS_STR_DICT, gstr, nulls=ng)]
        truth += [with_nulls(gint, ng), with_nulls(gstr, ng)]
        types += [OBJ_INT, OBJ_VARCHAR]
    else:
        group_cols = dict(GROUP_COLS_PAX)
        runs = np.repeat(rng.integers(0, 9, size=n // 10 + 1), 10)[:n] * 77
        gc = [7] * n
        for i in range(3, n, 41):
            gc[i] = int(gkey[i])
        cols += [ob.Column(OBJ_INT, ENC_DICT, as_store(gint), nulls=ng), ob.Column(OBJ_VARCHAR, ENC_DICT, gstr, nulls=ng),
                 ob.Column(OBJ_INT, ENC_RLE, as_store(runs.tolist())), ob.Column(OBJ_INT, ENC_CONST, as_store(gc))]
        truth += [with_nulls(gint, ng), with_nulls(gstr, ng), [int(x) for x in runs.tolist()], gc]
        types += [OBJ_INT, OBJ_VARCHAR, OBJ_INT, OBJ_INT]
    return Spec(cols, truth, rpb, group_cols, types, shape)


@functools.lru_cache(maxsize=None)
def matrix_table(tname, codec):
    import oceanbase_b200 as ob
    s = matrix_spec(tname, codec)
    return ob.encode_table(s.cols, s.rpb)


# ---- the reference fold --------------------------------------------------------------------------------------------
def fold(kind, a, b=None):
    """aggregate `kind` over the cells a (and b for SUM_PRODUCT): Python ints or None per row"""
    if kind == COUNT:
        return sum(1 for x in a if x is not None)
    if kind == SUM:
        return wrap128(sum(x for x in a if x is not None))
    if kind == SUM_PRODUCT:
        return wrap128(sum(x * y for x, y in zip(a, b) if x is not None and y is not None))
    live = [x for x in a if x is not None]
    if not live:
        return None
    return min(live) if kind == MIN else max(live)


def exact_group_by_model(blk, group_col, rows, aggs, cells):
    """Pushdown GROUP BY of one block as int64 [n_aggs][distinct count + 1][2] (the layout obgpu_block_group_by fills):
    group = the oracle's dictionary ref of the row (distinct count: the NULL group); cells[col][row]: the true value of a
    block cell (Python int or None). COUNT: (count, 0); SUM: the low and high words of the signed 128-bit sum; MIN / MAX:
    (the 64-bit image of the value as int64, 1), (0, 0) for a group without a non-NULL value. Unsigned 64-bit values keep
    their order and are zero-extended in sums."""
    rows = np.asarray(rows, dtype=np.int32)
    refs = blk.dict_refs(group_col, rows) if len(rows) else np.zeros(0, dtype=np.uint32)
    n_groups = blk.dict_count(group_col) + 1
    members = [[] for _ in range(n_groups)]
    for r, ref in zip(rows.tolist(), refs.tolist()):
        members[ref].append(r)
    out = np.zeros((len(aggs), n_groups, 2), dtype=np.int64)
    for k, (kind, col) in enumerate(aggs):
        for g in range(n_groups):
            if kind == COUNT and col < 0:
                out[k, g] = (len(members[g]), 0)
                continue
            got = fold(kind, [cells[col][r] for r in members[g]])
            if kind == COUNT:
                out[k, g] = (got, 0)
            elif kind == SUM:
                out[k, g] = (to_i64(got), to_i64(got >> 64))
            elif got is not None:
                out[k, g] = (to_i64(got), 1)
    return out


def block_cells(spec, b):
    """true values of block b's cells: {store col: list per block row}"""
    r0 = b * spec.rpb
    r1 = min(r0 + spec.rpb, spec.n)
    return {c: spec.truth[c][r0:r1] for c in range(len(spec.truth))}


# ---- what the oracle sees ------------------------------------------------------------------------------------------
def oracle_value(obj_type, cell):
    """the oracle's cell (64-bit image, bytes or None) as the column's own value"""
    if cell is None or isinstance(cell, bytes):
        return cell
    bits = 8 * datum_len(obj_type)
    v = int(cell) & ((1 << bits) - 1)
    signed = obj_type in (1, 2, 3, 4, 5, 17, 18, 19, 20)
    return v - (1 << bits) if signed and v >= 1 << (bits - 1) else v


def header_types(table, n_cols):
    """(set of codec ids per column over every block, CONST blocks with exceptions per column, CONST blocks without)"""
    img, off = np.asarray(table.image), np.asarray(table.offsets)
    kinds = [set() for _ in range(n_cols)]
    const_exc, const_plain = [0] * n_cols, [0] * n_cols
    for b in range(table.n_blocks):
        o = int(off[b])
        hs = int(img[o + 4:o + 8].view(np.uint32)[0])
        cs = int(img[o + 20]) == 3
        for c in range(n_cols):
            if cs:
                kinds[c].add(int(img[o + hs + 12 + 4 * c + 1]))
                continue
            h = img[o + hs + 16 * c:o + hs + 16 * c + 16]
            kinds[c].add(int(h[1]))
            if h[1] == ENC_CONST:
                meta = o + hs + 16 * n_cols + int(h[8:12].view(np.uint32)[0])
                if img[meta + 1] > 0:
                    const_exc[c] += 1
                else:
                    const_plain[c] += 1
    return kinds, const_exc, const_plain


def brute_fold(kind, a, b=None):
    """the same fold done the way a device does it: 64-bit words, explicit carries, order keys with the sign bit flipped"""
    lo = hi = 0
    seen = False
    for i, x in enumerate(a):
        if x is None or (kind == SUM_PRODUCT and b[i] is None):
            continue
        if kind == COUNT:
            lo += 1
            continue
        if kind in (SUM, SUM_PRODUCT):
            p = (x * b[i]) % M128 if kind == SUM_PRODUCT else x % M128
            nlo = lo + (p & (M64 - 1))
            hi = (hi + (p >> 64) + (nlo >> 64)) & (M64 - 1)
            lo = nlo & (M64 - 1)
            continue
        if not seen or (x < lo if kind == MIN else x > lo):
            lo, seen = x, True
    if kind == COUNT:
        return lo
    if kind in (SUM, SUM_PRODUCT):
        v = (hi << 64) | lo
        return v - M128 if hi >> 63 else v
    return lo if seen else None


MATRIX = [(t, c) for t in TYPES for c in CODECS]


@pytest.mark.parametrize("tname,codec", MATRIX)
def test_matrix_table_inputs_and_reference_fold(tname, codec):
    spec = matrix_spec(tname, codec)
    table = matrix_table(tname, codec)
    obj, lo, hi = TYPES[tname]
    enc = CODECS[codec][0]
    n_cols = len(spec.cols)
    # the oracle decodes every cell back to the generated value / NULL
    seen = set()
    for b in range(table.n_blocks):
        blk = ora.Block(table.block(b))
        cells = block_cells(spec, b)
        for c in range(n_cols):
            got = [oracle_value(spec.obj_types[c], blk.cell(c, r)) for r in range(blk.row_count)]
            assert got == cells[c], (tname, codec, b, c)
        seen.update(x for x in cells[VA] + cells[VB] if x is not None)
    for v in specials(tname):
        assert v in seen or CODECS[codec][2] in ("const", "runs"), (tname, codec, v)
    assert lo in seen or hi in seen
    # the codec the writer really chose, block by block
    kinds, const_exc, const_plain = header_types(table, n_cols)
    for c in (VA, VB, VN):
        assert kinds[c] == {HEADER_TYPE[vn_encoding(enc) if c == VN else enc]}, (tname, codec, c, kinds[c])
    for c, gc in spec.group_cols.items():
        want = {"dict_int": ENC_DICT, "dict_str": ENC_DICT, "rle": ENC_RLE, "const": ENC_CONST, "cs_int_dict": ENC_CS_INT_DICT,
                "cs_str_dict": ENC_CS_STR_DICT}[c]
        assert kinds[gc] == {HEADER_TYPE[want]}, (c, kinds[gc])
    if codec == "const":
        assert const_plain[VA] == table.n_blocks and const_exc[VB] == table.n_blocks
    if codec == "const_exc":
        assert const_exc[VA] == table.n_blocks
    if not is_cs(codec):
        assert const_exc[GROUP_COLS_PAX["const"]] == table.n_blocks
    # the reference fold == the word-wise fold over the oracle's cells
    for kind in (COUNT, SUM, MIN, MAX):
        for c in (W, VA, VB, VN):
            assert fold(kind, spec.truth[c]) == brute_fold(kind, spec.truth[c]), (kind, c)
    for a, b in ((VA, W), (VB, W), (VA, VB), (W, W), (VN, W)):
        assert fold(SUM_PRODUCT, spec.truth[a], spec.truth[b]) == brute_fold(SUM_PRODUCT, spec.truth[a], spec.truth[b])
    assert fold(MIN, spec.truth[VN]) is None and fold(SUM, spec.truth[VN]) == 0 and fold(COUNT, spec.truth[VN]) == 0
    # the value distributions reach what the device folds must survive
    if tname == "int":       # SUM past 2^64 upward and downward
        assert sum(x for x in spec.truth[VA]) >= M64 and sum(x for x in spec.truth[VB] if x is not None) <= -M64
    if tname == "uint64":
        assert sum(x for x in spec.truth[VA]) >= M64
    wsq = sum(x * x for x in spec.truth[W] if x is not None)
    assert wsq >= 1 << 127 and fold(SUM_PRODUCT, spec.truth[W], spec.truth[W]) != wsq      # INT64_MIN^2 rows wrap 2^127


def test_exact_group_by_model_orders_and_sums_unsigned_64bit():
    class FakeBlock:    # two groups + the NULL group
        def dict_refs(self, col, rows):
            return np.array([r % 3 for r in rows], dtype=np.uint32)

        def dict_count(self, col):
            return 2

    cells = {1: [M64 - 1, 5, None, 1 << 63, 7, 9]}
    out = exact_group_by_model(FakeBlock(), 0, np.arange(6), [(SUM, 1), (MIN, 1), (MAX, 1), (COUNT, 1), (COUNT, -1)], cells)
    s0 = (M64 - 1) + (1 << 63)        # rows 0 and 3: past 2^64, never negative
    assert (int(out[0, 0, 0]) % M64) + (int(out[0, 0, 1]) % M64 << 64) == s0
    assert int(out[1, 0, 0]) % M64 == 1 << 63 and int(out[2, 0, 0]) % M64 == M64 - 1      # unsigned order
    assert tuple(out[1, 2]) == (9, 1) and tuple(out[3, 2]) == (1, 0) and tuple(out[4, 2]) == (2, 0)     # NULL skipped
    cells = {1: [None] * 6}
    out = exact_group_by_model(FakeBlock(), 0, np.arange(6), [(SUM, 1), (MIN, 1), (COUNT, 1)], cells)
    assert not out.any()
