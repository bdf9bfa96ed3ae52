"""The tables tests/test_gpu_group_by_columns.py puts at each side of each limit of obgpu_result_group_by_columns, built here on
the CPU, and proof that each case sits where it claims.

The fold path of a GROUP BY over group columns c_0..c_{n-1} is chosen from P = prod (n_keys_c + 1), n_keys_c the distinct values
of column c in its dictionaries over the batch (group_values.cuh): CTA-private shared accumulators when
P x (n_aggs + 1) x 16 bytes <= kSharedAccBudget (48 KiB), global ones indexed by the composite id when P <= kDenseGroups (2^20),
and the hashed path otherwise, which refuses more than kHashGroups (2^22) distinct tuples among the selected rows. P of 2^64 - 1
or more is refused. The distinct counts are read from the block bytes through the oracle (oracle_binding.Block's dictionaries);
the distinct tuples come from the model cells. Also checked: the model's tuple order on hand-written tuples."""
import functools

import numpy as np
import pytest

import oracle_binding as ora
from test_scan_codes_model import CAP, cap_table

OBJ_INT, OBJ_UINT64 = 5, 10
ENC_RAW, ENC_DICT = 0, 1
SHARED_ACC_BUDGET = 48 << 10
DENSE_GROUPS = 1 << 20
HASH_GROUPS = 1 << 22
BIG_RPB = 2000


def tuple_order(t):
    """a group tuple's sort key: per column its value (ints in their own domain, bytes bytewise), NULL (None) last"""
    return tuple((v is None, 0 if v is None else v) for v in t)


def path_of(p, n_aggs):
    if p <= DENSE_GROUPS and p * (n_aggs + 1) * 16 <= SHARED_ACC_BUDGET:
        return "shared"
    return "global" if p <= DENSE_GROUPS else "hashed"


def dict_values(image, col, blocks=None):
    """the distinct dictionary entries of column col over the blocks (all by default), read through the oracle"""
    vals = set()
    for b in range(image.n_blocks) if blocks is None else blocks:
        blk = ora.Block(image.block(b))
        vals.update(blk.dict_entry(col, e)[0] for e in range(blk.dict_count(col)))
        ora.arena_reset()
    return vals


def int_table(cols, rpb, obj=OBJ_INT):
    import oceanbase_b200 as ob
    n = len(cols[0])
    return ob.encode_table([ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64))] +
                           [ob.Column(obj, ENC_DICT, np.asarray(c, dtype=np.int64)) for c in cols], rpb)


# ---- the tables -------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def shared_table():
    """0 row id; 1: 31 values; 2: 47; 3: 48. With one aggregate (COUNT(*): 2 accumulators), (1, 2) has P = 32 x 48 = 1536 and
    exactly 48 KiB of accumulators (shared); (1, 3) has P = 32 x 49 = 1568 (global)"""
    i = np.arange(4000)
    cells = [i % 31, i % 47, i % 48]
    return int_table(cells, 250), [i.tolist()] + [c.tolist() for c in cells]


@functools.lru_cache(maxsize=None)
def dense_table():
    """0 row id; 1, 2: 1023 values each, so (1, 2) has P = 2^20 (global); 3: 16 values, 4: 61 680 (every row its own), so (3, 4)
    has P = 17 x 61 681 = 2^20 + 1 (hashed). Blocks of 2000 rows: dictionaries larger than a warp's rank array"""
    i = np.arange(61_680)
    cells = [i % 1023, (i * 5) % 1023, i % 16, i]
    return int_table(cells, BIG_RPB), [i.tolist()] + [c.tolist() for c in cells]


@functools.lru_cache(maxsize=None)
def hash_cap_table():
    """0 row id; 1 a = i % 2048, 2 b = i // 2048 over 2^22 + 1 rows: every row a tuple of its own. Rows below 2^22 hold exactly
    kHashGroups tuples; all rows one more"""
    i = np.arange(HASH_GROUPS + 1, dtype=np.int64)
    return int_table([i % 2048, i // 2048], BIG_RPB), [i, i % 2048, i // 2048]


@functools.lru_cache(maxsize=None)
def carry_table():
    """0 m 0..99; 1 g1 (5 values), 2 g2 and 3 g3 (1000 values each in the first 3000 rows, then 3 and 2): P = 6 x 1001 x 1001
    (hashed) with 30 large groups; 4 INT near INT64_MAX, 5 UINT64 near 2^64 - 1: 128-bit sums over 2^22 + 12 345 rows"""
    import oceanbase_b200 as ob
    n = (1 << 22) + 12_345
    rng = np.random.default_rng(79)
    i = np.arange(n, dtype=np.int64)
    g1 = rng.integers(0, 5, n).astype(np.int64) * 1000 - 2000
    g2 = np.where(i < 3000, i % 1000, rng.integers(0, 3, n)).astype(np.int64) - 500
    g3 = np.where(i < 3000, (i * 7) % 1000, rng.integers(0, 2, n)).astype(np.int64)
    a = rng.integers(1 << 62, (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)
    a[rng.random(n) < 0.02] = np.iinfo(np.int64).min
    u = rng.integers(1 << 63, (1 << 64) - 1, size=n, dtype=np.uint64, endpoint=True)
    u[rng.integers(0, n, size=50)] = 0
    m = rng.integers(0, 100, n).astype(np.int64)
    cols = [ob.Column(OBJ_INT, ENC_RAW, m), ob.Column(OBJ_INT, ENC_DICT, g1), ob.Column(OBJ_INT, ENC_DICT, g2), ob.Column(OBJ_INT, ENC_DICT, g3),
            ob.Column(OBJ_INT, ENC_RAW, a), ob.Column(OBJ_UINT64, ENC_RAW, u.view(np.int64))]
    return ob.encode_table(cols, BIG_RPB), [m, g1, g2, g3, a, u]


# ---- each case at its side of its limit ------------------------------------------------------------------------------------
def test_shared_budget_sides():
    image, cells = shared_table()
    n = [len(dict_values(image, c)) for c in (1, 2, 3)]
    assert n == [31, 47, 48]
    assert (n[0] + 1) * (n[1] + 1) * 2 * 16 == SHARED_ACC_BUDGET and path_of((n[0] + 1) * (n[1] + 1), 1) == "shared"
    assert (n[0] + 1) * (n[2] + 1) * 2 * 16 > SHARED_ACC_BUDGET and path_of((n[0] + 1) * (n[2] + 1), 1) == "global"


def test_dense_limit_sides():
    image, cells = dense_table()
    n = [len(dict_values(image, c)) for c in (1, 2, 3, 4)]
    assert n == [1023, 1023, 16, 61_680]
    assert (n[0] + 1) * (n[1] + 1) == DENSE_GROUPS and path_of(DENSE_GROUPS, 1) == "global"
    assert (n[2] + 1) * (n[3] + 1) == DENSE_GROUPS + 1 and path_of(DENSE_GROUPS + 1, 1) == "hashed"
    assert max(ora.Block(image.block(b)).dict_count(1) for b in range(image.n_blocks)) > 256   # ranks probed per row
    ora.arena_reset()


def test_hash_cap_sides():
    image, (i, a, b) = hash_cap_table()
    na = len(dict_values(image, 1, blocks=range(2)))          # a lower bound: the first 4000 rows hold every value of a
    nb = len(dict_values(image, 2))
    assert na == 2048 and nb == 2049 and (na + 1) * (nb + 1) > DENSE_GROUPS
    below = np.unique(a[:HASH_GROUPS] * 4096 + b[:HASH_GROUPS]).size
    assert below == HASH_GROUPS and np.unique(a * 4096 + b).size == HASH_GROUPS + 1


def test_p_overflow_sides():
    t = cap_table()
    n = len(dict_values(t.image, 1))
    assert n == CAP and None not in t.cells[1]
    g = n + 1
    assert g ** 4 >= (1 << 64) - 1                         # named four times: refused
    assert g ** 3 < (1 << 64) - 1 and g ** 3 > DENSE_GROUPS
    top = (n - 1) * (g * g + g + 1)                         # the largest id of (v, v, v)
    assert top >= 1 << 48


def test_carry_table_is_hashed_with_carries():
    image, (m, g1, g2, g3, a, u) = carry_table()
    n = [len(dict_values(image, c)) for c in (1, 2, 3)]
    assert n == [5, 1000, 1000]
    assert (n[0] + 1) * (n[1] + 1) * (n[2] + 1) > DENSE_GROUPS
    big = (g1 * 1_000_000 + (g2 + 500) * 1000 + g3)[3000:]
    _, counts = np.unique(big, return_counts=True)
    assert counts.size == 30 and int(counts.min()) * (1 << 62) >= 1 << 64    # every large group's SUM(a) carries


def test_model_order_on_hand_written_tuples():
    tuples = [(None, b"a"), (1, None), (1, b""), (-5, b"\x80"), (1, b"a"), (None, None), (-5, b"\x00b"), (1, b"\x00"), (-5, None)]
    want = [(-5, b"\x00b"), (-5, b"\x80"), (-5, None), (1, b""), (1, b"\x00"), (1, b"a"), (1, None), (None, b"a"), (None, None)]
    assert sorted(tuples, key=tuple_order) == want
    u = [(1 << 64) - 1, 0, 1 << 63]        # an unsigned column: its own domain
    assert sorted([(x, 0) for x in u], key=tuple_order) == [(0, 0), (1 << 63, 0), ((1 << 64) - 1, 0)]


@pytest.mark.parametrize("p,n_aggs,want", [(1536, 1, "shared"), (1537, 1, "global"), (1024, 2, "shared"), (1025, 2, "global"),
                                           (DENSE_GROUPS, 16, "global"), (DENSE_GROUPS + 1, 1, "hashed")])
def test_path_rule(p, n_aggs, want):
    assert path_of(p, n_aggs) == want
