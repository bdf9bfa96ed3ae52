"""Column-group tables and the plain row-set model that tests/test_gpu_cg_bitmap_exact.py checks the device against.

A column-store table keeps every column group as its own SSTable with its own micro-block boundaries. Filter results of some
groups are folded into one range bitmap (obgpu_cg_bitmap_apply_result: set / and / or at a row offset), and other groups are
projected under it (obgpu_scan_bitmap). Here every column is its own group, written by encode_table at 1, 31, 33, 133, 500, 1025
or 2000 rows per block (each with a ragged last block; 133 = 5 mod 32, so 32 consecutive 133-row blocks start at every bit of a
word). The model of a filter is a bool array over the group's rows, built from the oracle's filter per block; a fold is plain
slicing at the row offset; a projection is the oracle's cells at the set bits.

CPU checks: every group's header shows the intended codec; the oracle's cells are the generated values; every filter's oracle
selection equals a numpy predicate on the generated values; the fold plans the GPU file runs reach every bit position of a word
for every fold op, share a seam word between two batches and cover n_rows % 32 of 0, 1 and 31, with and without all_true."""
import functools

import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import as_store, header_types, oracle_value

N = 133 * 33 + 71                     # rows of every column group: 34 blocks of 133, the last one 71 rows
RPBS = (1, 31, 33, 133, 500, 1025, 2000)
EQ, LE, LT, GE, GT, NE, BT, IN, NU, NN = range(10)     # OBGPU_WHITE_OP_*
OBJ = {"tinyint": 1, "int": 5, "uint64": 10, "date": 19, "varchar": 22}
ENC_RAW, ENC_DICT, ENC_STRING_DIFF, ENC_HEX = 0, 1, 5, 6
ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STR_DICT, ENC_AUTO = 16, 17, 19, 32
WORDS = [b"w%03d" % i + b"x" * (i % 13) for i in range(200)]
HEX_ALPHA = bytes([0x00, 0x80, 0xFF, 0x7F, 0x01, 0x41, 0x81, 0xC1]) + b"abcdefgh"

# column kind -> (object type, encoding, header codec ids the writer must leave in every block (None: checked apart))
KINDS = {
    "int_dict": ("int", ENC_DICT, {1}),             # sorted values: the skip index settles whole blocks
    "int_raw_null": ("int", ENC_RAW, {0}),
    "tiny_dict": ("tinyint", ENC_DICT, {1}),        # negative values: the sign fix of a one-byte store
    "u64_raw": ("uint64", ENC_RAW, {0}),            # values >= 2^63
    "date_raw": ("date", ENC_RAW, {0}),             # four-byte datums
    "int_auto": ("int", ENC_AUTO, None),            # one value in every other 133-row run: RLE / CONST there, DICT elsewhere
    "vc_dict": ("varchar", ENC_DICT, {1}),
    "vc_raw": ("varchar", ENC_RAW, {0}),
    "cs_int": ("int", ENC_CS_INTEGER, {0}),
    "cs_int_dict": ("int", ENC_CS_INT_DICT, {2}),
    "cs_str_dict": ("varchar", ENC_CS_STR_DICT, {3}),
    "vc_hex": ("varchar", ENC_HEX, {ENC_HEX}),      # strings the device rebuilds at open
}
STRING_KINDS = {k for k, v in KINDS.items() if v[0] == "varchar"}

# the groups: every kind at the small-block shape (133) and above the small-block limit (2000); the filter kinds at the other
# block sizes (a one-row block cannot hold a dictionary whose only cell is NULL, so only NULL-free kinds take rpb 1)
GROUPS = sorted({(k, r) for k in KINDS for r in (133, 2000)} | {("int_dict", r) for r in RPBS} |
                {("int_raw_null", r) for r in (31, 33, 500, 1025)} | {("vc_dict", r) for r in (31, 500)})


def with_nulls(values, mask):
    return [None if m else v for v, m in zip(values, mask.tolist())]


@functools.lru_cache(maxsize=None)
def values(kind):
    """the generated cells of a kind (Python ints / bytes, None for NULL), the same for every block size"""
    rng = np.random.default_rng(list(KINDS).index(kind) + 31)
    if kind == "int_dict":
        return [int(x) * 1_000_003 for x in np.sort(rng.integers(-400, 400, size=N))]
    if kind == "int_raw_null":
        v = [int(x) for x in rng.integers(-(1 << 40), 1 << 40, size=N)]
        v[:4] = [-(1 << 63), (1 << 63) - 1, 0, -1]
        return with_nulls(v, (rng.random(N) < 0.07).astype(np.uint8))
    if kind == "tiny_dict":
        return [int(x) for x in rng.integers(-128, 128, size=N)]
    if kind == "u64_raw":
        v = [int(x) for x in rng.integers(0, 1 << 63, size=N, dtype=np.uint64)]
        top = rng.random(N) < 0.5
        v = [x | (1 << 63) if t else x for x, t in zip(v, top.tolist())]
        v[:4] = [0, (1 << 64) - 1, 1 << 63, (1 << 63) - 1]
        return v
    if kind == "date_raw":
        v = [int(x) for x in rng.integers(-(1 << 31), 1 << 31, size=N)]
        v[:2] = [-(1 << 31), (1 << 31) - 1]
        return v
    if kind == "int_auto":
        v = rng.integers(0, 50, size=N)
        for b0 in range(0, N, 2 * 133):
            v[b0:b0 + 133] = 7
        return [int(x) for x in v]
    if kind == "vc_dict":
        return with_nulls([WORDS[i] for i in rng.integers(0, len(WORDS), size=N)], (rng.random(N) < 0.05).astype(np.uint8))
    if kind == "vc_raw":
        return [bytes(rng.integers(0, 256, size=int(rng.integers(0, 41)), dtype=np.uint8)) for _ in range(N)]
    if kind == "cs_int":
        return [int(x) for x in rng.integers(-10 ** 12, 10 ** 12, size=N)]
    if kind == "cs_int_dict":
        return [int(x) * 7 - 900 for x in rng.integers(0, 300, size=N)]
    if kind == "cs_str_dict":
        return [b"cs%03d" % x + b"q" * (x % 9) for x in rng.integers(0, 60, size=N)]
    if kind == "vc_hex":
        a = np.frombuffer(HEX_ALPHA, dtype=np.uint8)
        return [bytes(a[rng.integers(0, 16, size=int(rng.integers(0, 33)))]) for _ in range(N)]
    raise KeyError(kind)


def column(kind):
    import oceanbase_b200 as ob
    tname, enc, _ = KINDS[kind]
    v = values(kind)
    nulls = np.array([x is None for x in v], dtype=np.uint8)
    if tname == "varchar":
        return ob.Column(OBJ[tname], enc, [b"" if x is None else x for x in v], nulls=nulls if nulls.any() else None)
    return ob.Column(OBJ[tname], enc, as_store([0 if x is None else x for x in v]), nulls=nulls if nulls.any() else None)


@functools.lru_cache(maxsize=None)
def group_table(kind, rpb):
    import oceanbase_b200 as ob
    return ob.encode_table([column(kind)], rpb)


def block_starts(rpb):
    """first global row of every block of a group, and N behind the last"""
    return np.append(np.arange(0, N, rpb, dtype=np.int64), N)


@functools.lru_cache(maxsize=None)
def group_blocks(kind, rpb):
    t = group_table(kind, rpb)
    return [ora.Block(t.block(b)) for b in range(t.n_blocks)]


@functools.lru_cache(maxsize=None)
def cells(kind, rpb):
    """the oracle's cells of the group, as the column's own values (None for NULL)"""
    obj = OBJ[KINDS[kind][0]]
    if kind in STRING_KINDS:
        return [blk.cell(0, r) for blk in group_blocks(kind, rpb) for r in range(blk.row_count)]
    vals, isnull = ora.decode_column_ext(group_table(kind, rpb), 0)
    return [None if z else oracle_value(obj, v) for v, z in zip(vals.tolist(), isnull.tolist())]


# ---- filters: name -> (white filter leaf (op, params), predicate on one cell) -------------------------------------------
def _cmp(op, c):
    return {EQ: lambda x: x is not None and x == c, LE: lambda x: x is not None and x <= c, LT: lambda x: x is not None and x < c,
            GE: lambda x: x is not None and x >= c, GT: lambda x: x is not None and x > c, NE: lambda x: x is not None and x != c}[op]


FILTERS = {
    "int_dict": {"ge": (GE, (17 * 1_000_003,)), "bt": (BT, (-150 * 1_000_003, 90 * 1_000_003))},
    "int_raw_null": {"lt": (LT, (0,)), "nu": (NU, ())},
    "tiny_dict": {"ne": (NE, (-5,)), "lt": (LT, (0,))},
    "u64_raw": {"ge": (GE, (1 << 63,))},
    "date_raw": {"lt": (LT, (0,))},
    "int_auto": {"le": (LE, (20,))},
    "vc_dict": {"gt": (GT, (WORDS[100],)), "in": (IN, tuple(WORDS[k] for k in range(0, 200, 7))), "nn": (NN, ())},
    "vc_raw": {"ge": (GE, (b"\x80",))},
    "cs_int": {"gt": (GT, (0,))},
    "cs_int_dict": {"lt": (LT, (500,))},
    "cs_str_dict": {"in": (IN, (b"cs007qqqqqqq", b"cs040qqqq", b"cs059qqqqq"))},
    "vc_hex": {"ge": (GE, (b"a",))},
}


def white(kind, fname):
    import oceanbase_b200 as ob
    op, params = FILTERS[kind][fname]
    return ob.White(0, op, params)


def predicate(kind, fname):
    """numpy bool over the group's rows, from the generated values"""
    op, params = FILTERS[kind][fname]
    v = values(kind)
    if op == NU:
        return np.array([x is None for x in v])
    if op == NN:
        return np.array([x is not None for x in v])
    if op == BT:
        return np.array([x is not None and params[0] <= x <= params[1] for x in v])
    if op == IN:
        s = set(params)
        return np.array([x is not None and x in s for x in v])
    f = _cmp(op, params[0])
    return np.array([f(x) for x in v])


@functools.lru_cache(maxsize=None)
def selection(kind, rpb, fname):
    """the oracle's selection of a filter over the group's rows (None: no filter, every row)"""
    if fname is None:
        return np.ones(N, dtype=bool)
    flt = white(kind, fname)
    return np.concatenate([blk.filter_tree(flt).astype(bool) for blk in group_blocks(kind, rpb)])


def fold(bm, sel, row_offset, op):
    """obgpu_cg_bitmap_apply_result on the model: the batch's rows only, every other bit unchanged"""
    seg = bm[row_offset:row_offset + len(sel)]
    if op == "set":
        seg[:] = sel
    elif op == "and":
        seg &= sel
    else:
        seg |= sel
    return bm


# ---- fold plans ----------------------------------------------------------------------------------------------------------
# A step folds the result of one scan: (kind, rpb, filter name or None, count path, row offset, op). Count paths:
#   pipe0   OBGPU_PIPE=0: obgpu_count_kernel            rec     obgpu_count_pipe_kernel<true> (lean leaves, <= 512 rows)
#   plan    obgpu_count_pipe_kernel<false> (a string range leaf needs the plan's dictionary bitset)
#   big     OBGPU_PIPE=1 at 2000 rows per block: obgpu_count_pipe_kernel<false>
#   skip    aggregate rows attached: the skip index settles whole blocks always true / always false
#   all     no filter: the result has no words (all_selected)
#   capped  a filter-only scan with max_selected_rows=1: the fold is exact or refused, never partial
# Plans: (name, n_rows, all_true, steps). 2N = 24 mod 32, so 2N + 8 / 9 / 7 give n_rows % 32 of 0 / 1 / 31; a batch at N + k
# (k < 20) starts inside the word the batch at 0 ends in.
PLANS = [
    ("n0_all_true", 2 * N + 8, True, [
        ("int_dict", 133, "ge", "rec", 0, "and"),
        ("vc_dict", 133, "gt", "plan", N + 5, "or"),          # shares the seam word with the batch at 0
        ("int_raw_null", 33, "lt", "pipe0", 3, "and"),
        ("tiny_dict", 1025, None, "all", N + 8, "set"),
        ("int_dict", 31, "bt", "skip", 1, "or")]),
    ("n1_all_false", 2 * N + 9, False, [
        ("int_dict", 2000, "ge", "big", N + 9, "or"),
        ("int_dict", 500, "bt", "skip", 0, "or"),
        ("vc_dict", 500, "in", "pipe0", 0, "and"),
        ("int_raw_null", 1025, "lt", "capped", 17, "set"),
        ("int_dict", 33, "ge", "rec", N + 1, "and")]),
    ("n31_all_true", 2 * N + 7, True, [
        ("int_dict", 1, None, "all", 7, "and"),
        ("int_dict", 1, "ge", "rec", 7, "set"),
        ("vc_dict", 31, "gt", "plan", N + 7, "and"),
        ("int_raw_null", 31, "nu", "pipe0", N + 2, "or")]),
]
# every residue of the row offset: one group folded at offsets 0..31 in turn, the op cycling
SWEEP_ROWS = N + 40
SWEEP = [("int_dict", 500, "bt", "rec", off, ("set", "or", "and")[off % 3]) for off in range(32)]


def fold_steps():
    return [s for _, _, _, steps in PLANS for s in steps] + SWEEP


# ---- CPU checks ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,rpb", GROUPS, ids=[f"{k}-{r}" for k, r in GROUPS])
def test_group_headers_and_cells(kind, rpb):
    t = group_table(kind, rpb)
    assert t.total_rows == N and t.n_blocks == len(block_starts(rpb)) - 1
    assert [blk.row_count for blk in group_blocks(kind, rpb)] == np.diff(block_starts(rpb)).tolist()
    assert rpb == 1 or N % rpb != 0            # a ragged last block
    kinds = header_types(t, 1)[0][0]
    want = KINDS[kind][2]
    if want is not None:
        assert kinds == want, (kind, rpb, kinds)
    assert cells(kind, rpb) == values(kind)


def test_auto_column_takes_run_codecs_and_dictionaries():
    kinds = header_types(group_table("int_auto", 133), 1)[0][0]
    assert kinds & {2, 3} and kinds - {2, 3}, kinds


@pytest.mark.parametrize("kind,rpb", GROUPS, ids=[f"{k}-{r}" for k, r in GROUPS])
def test_oracle_selection_is_the_predicate(kind, rpb):
    for fname in FILTERS[kind]:
        sel = selection(kind, rpb, fname)
        assert np.array_equal(sel, predicate(kind, fname)), (kind, rpb, fname)
        assert 0 < sel.sum() < N, (kind, fname)


def test_values_reach_the_edges():
    assert any(x is not None and x >= 1 << 63 for x in values("u64_raw"))
    assert min(values("tiny_dict")) == -128 and max(values("tiny_dict")) == 127
    assert any(x is None for x in values("int_raw_null")) and any(x is None for x in values("vc_dict"))
    assert any(len(x) == 0 for x in values("vc_raw")) and any(len(x) > 32 for x in values("vc_raw"))


def test_fold_plans_reach_every_bit_position_and_seam():
    for op in ("set", "and", "or"):
        res = set()
        for kind, rpb, _, _, off, o in fold_steps():
            if o == op:
                res |= {int(x) % 32 for x in block_starts(rpb)[:-1] + off}
        assert res == set(range(32)), op
    assert {off % 32 for *_, off, _ in SWEEP} == set(range(32))
    assert {n % 32 for _, n, _, _ in PLANS} == {0, 1, 31}
    assert {t for _, _, t, _ in PLANS} == {True, False}
    for name, n_rows, _, steps in PLANS:
        offs = sorted({off for *_, off, _ in steps})
        assert all(off + N <= n_rows for off in offs), name
        # two batches side by side: the first ends inside a word the second starts in
        assert any(N // 32 == b // 32 and b >= N for b in offs), name
    assert {s[3] for s in fold_steps()} == {"pipe0", "rec", "plan", "big", "skip", "all", "capped"}


def test_fold_model_is_slicing():
    rng = np.random.default_rng(5)
    bm = rng.random(100) < 0.5
    sel = rng.random(37) < 0.5
    for op in ("set", "and", "or"):
        got = fold(bm.copy(), sel, 29, op)
        assert np.array_equal(got[:29], bm[:29]) and np.array_equal(got[66:], bm[66:])
        want = {"set": sel, "and": bm[29:66] & sel, "or": bm[29:66] | sel}[op]
        assert np.array_equal(got[29:66], want)
