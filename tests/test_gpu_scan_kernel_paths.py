"""Every branch of the small-block pipelined scan kernels (scan_small.cuh) against the oracle, with the pipelined
kernels forced on (OBGPU_PIPE=1) and off (OBGPU_PIPE=0): selected rows, row ids, every projected column, lengths and
NULLs must not depend on which kernels ran."""
import numpy as np
import pytest

import oracle_binding as ora
from test_gpu_scan import assert_scan_matches

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


class W:
    def __init__(self, table, flt, proj, is_str, elem):
        self.table, self.filter, self.proj, self.proj_is_string, self.proj_elem_len = table, flt, proj, is_str, elem


def pax_table(ob, n, rpb, seed):
    """c0 INT DICT (sorted dictionary), c1 VARCHAR DICT (1000 entries, some NULL), c2 INT RLE, c3 narrow INT RAW,
    c4 VARCHAR DICT with few entries, c5 INT RAW with NULLs."""
    rng = np.random.default_rng(seed)
    c0 = rng.integers(-300, 300, size=n, dtype=np.int64) * 1_000_003
    words = [b"w%05d" % i + b"x" * (i % 13) for i in range(1000)]
    r1 = rng.integers(0, len(words), size=n)
    s1 = [words[i] for i in r1]
    n1 = (rng.random(n) < 0.03).astype(np.uint8)
    c2 = np.repeat(rng.integers(-5, 5, size=n // 40 + 1, dtype=np.int64) * 7_777_777_777, 40)[:n]
    c3 = rng.integers(0, 200, size=n, dtype=np.int64)
    few = [b"alpha", b"beta", b"gamma-long-string-value", b"delta"]
    s4 = [few[i] for i in rng.integers(0, len(few), size=n)]
    c5 = rng.integers(-1000, 1000, size=n, dtype=np.int64)
    n5 = (rng.random(n) < 0.05).astype(np.uint8)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_DICT, c0), ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s1, nulls=n1),
            ob.Column(ob.OBJ_INT, ob.ENC_RLE, c2), ob.Column(ob.OBJ_INT, ob.ENC_RAW, c3),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s4), ob.Column(ob.OBJ_INT, ob.ENC_RAW, c5, nulls=n5)]
    return ob.encode_table(cols, rpb), words, few


PROJ = [0, 1, 2, 4, 5]
PROJ_STR = [False, True, False, True, False]
PROJ_LEN = [8, 8, 8, 8, 8]


def filters(ob, words, few):
    Wt = ob.White
    in_hashable = tuple(words[k] for k in (3, 50, 400, 777))
    in_unhashable = tuple(words[k] for k in range(0, 1000, 25))   # 40 constants: more than the host's hash slots take
    return {
        "sorted_int_range": Wt(0, ob.WHITE_OP_BT, (-100 * 1_000_003, 50 * 1_000_003)),
        "sorted_int_range_ne_and": ob.And([Wt(0, ob.WHITE_OP_GE, (-250 * 1_000_003,)), Wt(3, ob.WHITE_OP_LT, (150,))]),
        "str_eq_first": Wt(1, ob.WHITE_OP_EQ, (words[17],)),
        "str_ne_first": Wt(1, ob.WHITE_OP_NE, (words[17],)),
        "str_in_first": Wt(1, ob.WHITE_OP_IN, in_hashable),
        "str_in_unhashable": Wt(1, ob.WHITE_OP_IN, in_unhashable),
        "str_in_or": ob.Or([Wt(3, ob.WHITE_OP_LT, (5,)), Wt(1, ob.WHITE_OP_IN, in_hashable), Wt(4, ob.WHITE_OP_EQ, (few[2],))]),
        "str_eq_or_unhashable": ob.Or([Wt(1, ob.WHITE_OP_IN, in_unhashable), Wt(4, ob.WHITE_OP_NE, (few[0],))]),
        "survivor_str": ob.And([Wt(3, ob.WHITE_OP_LT, (3,)), Wt(1, ob.WHITE_OP_IN, in_hashable + (words[5],))]),
        "survivor_str_ne": ob.And([Wt(0, ob.WHITE_OP_EQ, (7 * 1_000_003,)), Wt(1, ob.WHITE_OP_NE, (words[9],))]),
        "survivor_str_gt": ob.And([Wt(3, ob.WHITE_OP_EQ, (11,)), Wt(1, ob.WHITE_OP_GT, (words[500],))]),
        "non_dict_leaf": ob.And([Wt(5, ob.WHITE_OP_GT, (-500,)), Wt(2, ob.WHITE_OP_LE, (0,)), Wt(4, ob.WHITE_OP_IN, (few[1], few[3]))]),
        "rle_leaf_or": ob.Or([Wt(2, ob.WHITE_OP_EQ, (3 * 7_777_777_777,)), Wt(5, ob.WHITE_OP_NU, ())]),
        "all_rows": Wt(3, ob.WHITE_OP_GE, (0,)),
    }


@pytest.mark.parametrize("rpb,n", [(133, 12_000), (1100, 20_000)])
@pytest.mark.parametrize("case", ["sorted_int_range", "sorted_int_range_ne_and", "str_eq_first", "str_ne_first", "str_in_first",
                                  "str_in_unhashable", "str_in_or", "str_eq_or_unhashable", "survivor_str", "survivor_str_ne",
                                  "survivor_str_gt", "non_dict_leaf", "rle_leaf_or", "all_rows"])
def test_pax_leaves_and_projection(ob, ctx, pipe, rpb, n, case):
    table, words, few = pax_table(ob, n, rpb, seed=rpb)
    flt = filters(ob, words, few)[case]
    assert_scan_matches(ctx, W(table, flt, PROJ, PROJ_STR, PROJ_LEN))


def test_unsorted_int_dictionary_range(ob, ctx, pipe):
    # CS INT_DICT dictionaries are not sorted and carry a base: the range leaf goes through the predicate bitset
    rng = np.random.default_rng(21)
    n = 8000
    k = rng.integers(0, 300, size=n, dtype=np.int64) * 1001 + 5_000_000
    v = rng.integers(-20, 20, size=n, dtype=np.int64)
    s = [b"s%03d" % x for x in rng.integers(0, 40, size=n)]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_CS_INT_DICT, k), ob.Column(ob.OBJ_INT, ob.ENC_CS_INTEGER, v),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_CS_STR_DICT, s)]
    table = ob.encode_table(cols, 133)
    for flt in (ob.White(0, ob.WHITE_OP_BT, (5_000_000 + 1001 * 20, 5_000_000 + 1001 * 200)),
                ob.And([ob.White(0, ob.WHITE_OP_LT, (5_000_000 + 1001 * 150,)), ob.White(1, ob.WHITE_OP_GE, (0,))])):
        assert_scan_matches(ctx, W(table, flt, [0, 1, 2], [False, False, True], [8, 8, 8]))


def test_large_blocks_with_narrow_filter_columns(ob, ctx, pipe):
    # blocks of 2000 rows: more than 32 bitmap words. The pipelined count kernel takes a scan only when every filter
    # column's region is at most 12288 bytes (layout_pipe): a is dictionary-coded with 16 entries (a few bits per ref)
    # and b (0..99) is bit-packed by ENC_RAW to 7 bits per value, about 1.8 KB per block, so the scan stays eligible
    rng = np.random.default_rng(8)
    n = 16_000
    a = rng.integers(0, 16, size=n, dtype=np.int64)
    b = rng.integers(0, 100, size=n, dtype=np.int64)
    c = rng.integers(-10**12, 10**12, size=n, dtype=np.int64)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_DICT, a), ob.Column(ob.OBJ_INT, ob.ENC_RAW, b), ob.Column(ob.OBJ_INT, ob.ENC_RAW, c)]
    table = ob.encode_table(cols, 2000)
    for flt in (ob.And([ob.White(0, ob.WHITE_OP_LT, (9,)), ob.White(1, ob.WHITE_OP_BT, (10, 70))]),
                ob.Or([ob.White(1, ob.WHITE_OP_LT, (5,)), ob.White(0, ob.WHITE_OP_EQ, (3,))])):
        assert_scan_matches(ctx, W(table, flt, [0, 1, 2], [False] * 3, [8] * 3))


def test_skip_index_decided_blocks(ob, ctx, pipe):
    rng = np.random.default_rng(5)
    n = 13_300
    k = np.sort(rng.integers(0, 1 << 30, size=n, dtype=np.int64))
    words = [b"v%04d" % i for i in range(300)]
    s = [words[i] for i in rng.integers(0, len(words), size=n)]
    v = rng.integers(0, 100, size=n, dtype=np.int64)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_INTEGER_BASE_DIFF, k), ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, v)]
    table = ob.encode_table(cols, 133)
    agg = ob.table_agg_rows(cols, [0, 1, 2], 133)
    for flt in (ob.White(0, ob.WHITE_OP_BT, (int(k[3000]), int(k[9000]))),
                ob.And([ob.White(0, ob.WHITE_OP_GE, (int(k[4000]),)), ob.White(1, ob.WHITE_OP_IN, (words[3], words[77]))])):
        assert_scan_matches(ctx, W(table, flt, [0, 1, 2], [False, True, False], [8, 8, 8]), agg=agg)
