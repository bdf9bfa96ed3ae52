"""The tables tests/test_gpu_top_rows.py sorts hold what its cases claim, proved on the CPU from the block bytes.

- The k-limit table decodes, through the oracle, back to its model. It has more than 65 536 rows, one all-equal key column,
  a 16-value DICT key column (so the 1000th and the 65 536th row fall inside a tie), and a VARCHAR DICT key whose 16 values
  share their first 8 bytes (so the order is decided past the first order word).
- The string pool behind the string matrix holds the byte orders a first-8-byte word cannot settle: the empty string, a proper
  prefix, "ab" next to "ab\\0", strings equal in their first 8 bytes, and bytes >= 0x80. Each string codec of the matrix really
  wrote its header type into every block.
- The integer matrix holds each type's extremes: INT64_MIN / MAX, UINT64_MAX, -1 where the type is signed."""
import functools

import numpy as np
import pytest

import oracle_binding as ora
import test_string_filter_exact as sfe
from test_aggregate_exact import TYPES, VA, matrix_spec, specials

BIG_ROWS, BIG_RPB = 70_000, 500


@functools.lru_cache(maxsize=None)
def big_table():
    """0 row id; 1 INT, every row 5 (RAW); 2 INT of 16 values (DICT); 3 VARCHAR of 16 values sharing 8 bytes (DICT)"""
    import oceanbase_b200 as ob
    n = BIG_ROWS
    rng = np.random.default_rng(31)
    v2 = rng.integers(-8, 8, n).astype(np.int64)
    s3 = [b"prefix08-%02d" % int(x) for x in rng.integers(0, 16, n)]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(ob.OBJ_INT, ob.ENC_RAW, np.full(n, 5, dtype=np.int64)),
            ob.Column(ob.OBJ_INT, ob.ENC_DICT, v2), ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s3)]
    return ob.encode_table(cols, BIG_RPB), [list(range(n)), [5] * n, v2.tolist(), s3]


def test_big_table():
    image, cells = big_table()
    assert image.n_blocks * BIG_RPB == BIG_ROWS > 65536
    r0 = 0
    for b in range(0, image.n_blocks, 7):       # every seventh block, through the oracle
        blk = ora.Block(image.block(b))
        r0 = b * BIG_RPB
        for c in range(4):
            want = cells[c][r0:r0 + blk.row_count]
            if c < 3:                            # the oracle gives an integer's 64-bit image
                want = [v & ((1 << 64) - 1) for v in want]
            got = [blk.cell(c, r) for r in range(blk.row_count)]
            assert [v & ((1 << 64) - 1) if c < 3 else v for v in got] == want, (b, c)
        assert blk.dict_count(2) <= 16 and blk.dict_count(3) <= 16
    ora.arena_reset()
    v2 = np.array(cells[2])
    assert len(set(cells[2])) == 16 and len(set(cells[3])) == 16 and len({s[:8] for s in cells[3]}) == 1
    srt = np.sort(v2)
    for k in (1000, 65536):                      # the k-th row sits inside a tie, with tied rows on both sides of it
        assert srt[k - 1] == srt[k] and (srt == srt[k - 1]).sum() > 2


def test_string_pool_edges():
    pool = set(sfe.EDGE)
    assert b"" in pool
    assert any(a != b and b.startswith(a) and len(a) > 0 for a in pool for b in pool)             # a proper prefix
    assert any(a + b"\x00" in pool for a in pool)                                                   # "ab" and "ab\0"
    assert any(a != b and a[:8] == b[:8] and len(a) >= 8 and len(b) >= 8 for a in pool for b in pool)
    assert any(any(x >= 0x80 for x in a) for a in pool)
    assert any(len(a) > 14 for a in pool)                                                           # past two order words


@pytest.mark.parametrize("codec", list(sfe.CODECS))
def test_string_codecs_in_headers(codec):
    spec = sfe.spec_of(codec, "varchar", "n10")
    table = sfe.table_of(codec, "varchar", "n10")
    want = sfe.CODECS[codec][2]
    assert all(f[0] == want for f in sfe.header_facts(table, sfe.S)), codec
    assert any(v is None for v in spec.truth[sfe.S])


@pytest.mark.parametrize("tname", list(TYPES))
def test_int_extremes(tname):
    spec = matrix_spec(tname, "raw")
    vals = set(v for v in spec.truth[VA] if v is not None)
    assert set(specials(tname)) <= vals, tname
