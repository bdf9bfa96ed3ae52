"""The small-block projection kernel's single pass over (column, selected row) items for flat columns (plain K_BITS, integer
dictionaries, variable-length string dictionaries) against the oracle, with the pipelined kernels forced on (OBGPU_PIPE=1) and
off (OBGPU_PIPE=0): flat columns next to per-column ones (ext bits, RLE, CONST, raw strings) in the same block, 1-byte outputs,
sign-extended dictionary entries, NULLs, every row selected, no row selected, and 1, 3, 133, 400 and 512 rows per block."""
import numpy as np
import pytest

from test_gpu_scan import assert_scan_matches
from test_gpu_scan_kernel_paths import W

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


@pytest.fixture(params=["1", "0"], ids=["pipe", "no_pipe"])
def pipe(request, monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", request.param)
    return request.param


WORDS = [b"k%04d" % i + b"z" * (i % 11) for i in range(600)]


def mixed_table(ob, n, rpb, seed):
    """Flat and per-column kinds side by side:
    c0 INT DICT with NULLs (sorted dictionary)   c1 VARCHAR DICT with NULLs      c2 INT RAW, bit-packed (plain K_BITS)
    c3 INT RAW with NULLs (ext bits)            c4 INT RLE                      c5 INT CONST with exceptions and NULLs
    c6 DATE DICT (4-byte datum)                 c7 VARCHAR RAW                  c8 INT32 RAW"""
    rng = np.random.default_rng(seed)
    row = np.arange(n)
    c0 = rng.integers(-40, 40, size=n, dtype=np.int64) * 1_000_000_007
    n0 = (rng.random(n) < 0.04).astype(np.uint8)
    s1 = [WORDS[i] for i in rng.integers(0, len(WORDS), size=n)]
    n1 = (rng.random(n) < 0.05).astype(np.uint8)
    c2 = rng.integers(0, 3000, size=n, dtype=np.int64)
    c3 = rng.integers(-(1 << 40), 1 << 40, size=n, dtype=np.int64)
    n3 = (rng.random(n) < 0.05).astype(np.uint8)
    c4 = np.repeat(rng.integers(-4, 4, size=n // 9 + 1, dtype=np.int64) * 123_456_789, 9)[:n]
    c5 = np.full(n, 777, dtype=np.int64)
    c5[row % 53 == 4] = -3
    n5 = (row % 71 == 9).astype(np.uint8)
    c6 = rng.integers(-20000, 20000, size=n, dtype=np.int64)
    s7 = [b"raw-%d" % (i % 37) for i in rng.integers(0, 1000, size=n)]
    c8 = rng.integers(-(1 << 31), 1 << 31, size=n, dtype=np.int64)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_DICT, c0, nulls=n0), ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s1, nulls=n1),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, c2), ob.Column(ob.OBJ_INT, ob.ENC_RAW, c3, nulls=n3),
            ob.Column(ob.OBJ_INT, ob.ENC_RLE, c4), ob.Column(ob.OBJ_INT, ob.ENC_CONST, c5, nulls=n5),
            ob.Column(ob.OBJ_DATE, ob.ENC_DICT, c6), ob.Column(ob.OBJ_VARCHAR, ob.ENC_RAW, s7),
            ob.Column(ob.OBJ_INT32, ob.ENC_RAW, c8)]
    return ob.encode_table(cols, rpb)


PROJ = [0, 1, 2, 3, 4, 5, 6, 7, 8]
IS_STR = [False, True, False, False, False, False, False, True, False]
ELEM = [8, 8, 8, 8, 8, 8, 4, 8, 8]
K = 1_000_000_007


def filters(ob):
    Wt = ob.White
    ins = tuple(WORDS[i] for i in (2, 99, 300, 451, 599))
    return {
        "none": None,
        "every_row": Wt(2, ob.WHITE_OP_GE, (0,)),
        "and_three_dict": ob.And([Wt(0, ob.WHITE_OP_LT, (20 * K,)), Wt(6, ob.WHITE_OP_GT, (-15000,)), Wt(1, ob.WHITE_OP_IN, ins)]),
        "and_first_kills": ob.And([Wt(0, ob.WHITE_OP_GT, (10**15,)), Wt(1, ob.WHITE_OP_IN, ins), Wt(6, ob.WHITE_OP_LT, (0,))]),
        "or_dict": ob.Or([Wt(0, ob.WHITE_OP_EQ, (3 * K,)), Wt(1, ob.WHITE_OP_EQ, (WORDS[7],)), Wt(6, ob.WHITE_OP_BT, (0, 400))]),
        "or_mixed": ob.Or([Wt(2, ob.WHITE_OP_LT, (40,)), Wt(1, ob.WHITE_OP_NE, (WORDS[5],)), Wt(0, ob.WHITE_OP_NU, ())]),
        "survivor_str": ob.And([Wt(2, ob.WHITE_OP_LT, (60,)), Wt(0, ob.WHITE_OP_NE, (5 * K,)), Wt(1, ob.WHITE_OP_IN, ins)]),
        "sorted_ne": ob.And([Wt(0, ob.WHITE_OP_NE, (-7 * K,)), Wt(1, ob.WHITE_OP_NE, (WORDS[1],))]),
        "sorted_ne_alone": Wt(0, ob.WHITE_OP_NE, (11 * K,)),
        "int_bitset_and_str": ob.And([Wt(6, ob.WHITE_OP_BT, (-5000, 9000)), Wt(1, ob.WHITE_OP_NE, (WORDS[3],)),
                                      Wt(0, ob.WHITE_OP_GE, (-30 * K,))]),
    }


@pytest.mark.parametrize("rpb,n", [(133, 9_000), (3, 600), (512, 6_000)])
@pytest.mark.parametrize("case", ["none", "every_row", "and_three_dict", "and_first_kills", "or_dict", "or_mixed", "survivor_str",
                                  "sorted_ne", "sorted_ne_alone", "int_bitset_and_str"])
def test_flat_and_per_column_projection(ob, ctx, pipe, rpb, n, case):
    table = mixed_table(ob, n, rpb, seed=rpb + 1)
    assert_scan_matches(ctx, W(table, filters(ob)[case], PROJ, IS_STR, ELEM))


def test_one_row_blocks(ob, ctx, pipe):
    rng = np.random.default_rng(6)
    n = 400
    cols = [ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, [WORDS[i] for i in rng.integers(0, 50, size=n)]),
            ob.Column(ob.OBJ_INT, ob.ENC_DICT, rng.integers(-9, 9, size=n, dtype=np.int64) * K),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 1000, size=n, dtype=np.int64))]
    table = ob.encode_table(cols, 1)
    for flt in (None, ob.White(2, ob.WHITE_OP_LT, (500,)), ob.And([ob.White(1, ob.WHITE_OP_GE, (0,)), ob.White(0, ob.WHITE_OP_NE, (WORDS[3],))])):
        assert_scan_matches(ctx, W(table, flt, [0, 1, 2], [True, False, False], [8, 8, 8]))


def test_many_flat_items_per_block(ob, ctx, pipe):
    # 12 flat columns x up to 400 selected rows per block: far more (column, row) items than one warp step covers
    rng = np.random.default_rng(4)
    n = 8_000
    cols, is_str = [], []
    for k in range(12):
        if k % 3 == 0:
            cols.append(ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, [WORDS[i] for i in rng.integers(0, 200 + k, size=n)],
                                  nulls=(rng.random(n) < 0.02).astype(np.uint8)))
        elif k % 3 == 1:
            cols.append(ob.Column(ob.OBJ_INT, ob.ENC_DICT, rng.integers(-100, 100, size=n, dtype=np.int64) * (k + 1) * 99991))
        else:
            cols.append(ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 1 << (5 * k), size=n, dtype=np.int64)))
        is_str.append(k % 3 == 0)
    table = ob.encode_table(cols, 400)
    for flt in (None, ob.White(2, ob.WHITE_OP_LT, (1 << 9,))):
        assert_scan_matches(ctx, W(table, flt, list(range(12)), is_str, [8] * 12))


def test_narrow_and_sign_fixed_flat_columns(ob, ctx, pipe):
    # 1-byte outputs (YEAR: raw bit-packed and dictionary) and integer dictionaries whose entries are sign-extended on load
    # (TINYINT / INT32 store sizes under 8 bytes: a nonzero int_mask on the flat entry)
    rng = np.random.default_rng(9)
    n = 6_000
    cols = [ob.Column(ob.capi.OBJ_YEAR, ob.ENC_RAW, rng.integers(0, 200, size=n, dtype=np.int64)),
            ob.Column(ob.capi.OBJ_YEAR, ob.ENC_DICT, rng.integers(0, 120, size=n, dtype=np.int64)),
            ob.Column(ob.OBJ_TINYINT, ob.ENC_DICT, rng.integers(-128, 128, size=n, dtype=np.int64),
                      nulls=(rng.random(n) < 0.03).astype(np.uint8)),
            ob.Column(ob.OBJ_INT32, ob.ENC_DICT, rng.integers(-(1 << 31), 1 << 31, size=n // 50, dtype=np.int64)[rng.integers(0, n // 50, size=n)]),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 1000, size=n, dtype=np.int64))]
    table = ob.encode_table(cols, 133)
    for flt in (None, ob.White(4, ob.WHITE_OP_LT, (300,)), ob.Or([ob.White(2, ob.WHITE_OP_LT, (-100,)), ob.White(3, ob.WHITE_OP_GT, (0,))])):
        assert_scan_matches(ctx, W(table, flt, [0, 1, 2, 3, 4], [False] * 5, [1, 1, 8, 8, 8]))
