"""The tables test_gpu_group_by_any and test_gpu_pipeline_group_by_any rely on, proved from the block bytes on the CPU: which
blocks of auto_table are not dictionary coded (so GROUP BY takes the cells path there), the distinct keys at both sides of
the cells fold's first capacity (2^20) and of the dictionary fold's value cap (65 536), that the contention table's key and
value columns are RAW in every block, and that its true 128-bit sums exceed 2^64."""
import functools

import numpy as np

from test_aggregate_exact import ENC_CONST, ENC_DICT, ENC_RAW, ENC_RLE, OBJ_INT
from test_scan_codes_model import CAP, auto_table, cap_table

OBJ_UINT64 = 10
FIRST_GROUPS = 1 << 20          # gcells::kFirstGroups
REFOLD_RPB = 4000
DICT_KINDS = {ENC_DICT, ENC_RLE, ENC_CONST}   # what the dictionary GROUP BY folds (is_dict_kind)


def block_codecs(image, col):
    """the ObColumnHeader::type_ of a PAX column in every block"""
    img, off = np.asarray(image.image), np.asarray(image.offsets)
    out = []
    for b in range(image.n_blocks):
        o = int(off[b])
        hs = int(img[o + 4:o + 8].view(np.uint32)[0])
        out.append(int(img[o + hs + 16 * col + 1]))
    return out


@functools.lru_cache(maxsize=None)
def refold_table():
    """0 row id; 1 a RAW INT key, distinct in rows 0..2^20 and 100 values after; 2 a RAW value. Rows below 2^20 hold 2^20
    keys (one fold), rows up to 2^20 one more (the refold)"""
    import oceanbase_b200 as ob
    n = FIRST_GROUPS + 1 + 3 * REFOLD_RPB
    i = np.arange(n, dtype=np.int64)
    key = np.where(i <= FIRST_GROUPS, i, i % 100) * 3 - 7
    val = (i * 7919) % 100_003 - 50_000
    cols = [ob.Column(OBJ_INT, ENC_RAW, i), ob.Column(OBJ_INT, ENC_RAW, key), ob.Column(OBJ_INT, ENC_RAW, val)]
    return ob.encode_table(cols, REFOLD_RPB), [i, key, val]


CONT_ROWS, CONT_RPB = 40_000, 2000


@functools.lru_cache(maxsize=None)
def contention_table():
    """0 row id; 1 one value in every row, 2 sixteen values, both RAW (the cells path, every lane of a warp on one or a few
    groups); 3 INT near INT64_MAX with INT64_MIN in 3 %; 4 UINT64 near 2^64; 5 INT at both extremes and 0"""
    import oceanbase_b200 as ob
    rng = np.random.default_rng(91)
    n = CONT_ROWS
    i = np.arange(n, dtype=np.int64)
    one = np.full(n, 42, dtype=np.int64)
    g16 = (i * 7 % 16) * 5 - 30
    a = rng.integers((1 << 63) - (1 << 40), (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)
    a[rng.random(n) < 0.03] = np.iinfo(np.int64).min
    u = rng.integers((1 << 64) - (1 << 40), (1 << 64) - 1, size=n, dtype=np.uint64, endpoint=True)
    e = rng.choice(np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0], dtype=np.int64), n)
    cols = [ob.Column(OBJ_INT, ENC_RAW, i), ob.Column(OBJ_INT, ENC_RAW, one), ob.Column(OBJ_INT, ENC_RAW, g16), ob.Column(OBJ_INT, ENC_RAW, a),
            ob.Column(OBJ_UINT64, ENC_RAW, u.view(np.int64)), ob.Column(OBJ_INT, ENC_RAW, e)]
    return ob.encode_table(cols, CONT_RPB), [i, one, g16, a, u, e]


def test_auto_table_mixes_dictionary_and_raw_blocks():
    t = auto_table()
    for col in (1, 2):
        codecs = block_codecs(t.image, col)
        raw = [b for b, c in enumerate(codecs) if c not in DICT_KINDS]
        assert raw and len(raw) < len(codecs), (col, codecs)
        assert all(b % 4 == 3 for b in raw), (col, codecs)
        assert all(codecs[b] in DICT_KINDS for b in range(3)), (col, codecs)   # the first three blocks: a dictionary-only batch
    assert set(block_codecs(t.image, 3)) == {ENC_DICT}


def test_refold_table_sides():
    image, (i, key, _) = refold_table()
    assert set(block_codecs(image, 1)) == {ENC_RAW}
    assert len(np.unique(key[i < FIRST_GROUPS])) == FIRST_GROUPS
    assert len(np.unique(key[i <= FIRST_GROUPS])) == FIRST_GROUPS + 1


def test_cap_table_sides():
    t = cap_table()
    assert len(set(t.cells[1])) == CAP and len(set(t.cells[2])) == CAP + 1


def test_contention_table_is_raw_and_sums_exceed_64_bits():
    image, (i, one, g16, a, u, e) = contention_table()
    for c in range(6):
        assert set(block_codecs(image, c)) == {ENC_RAW}, c
    assert len(np.unique(one)) == 1 and len(np.unique(g16)) == 16
    assert sum(int(x) for x in a) > 1 << 64
    assert sum(int(x) for x in u) > 1 << 64
    for g in np.unique(g16):   # every 16-value group too, so a warp's pre-reduction carries
        assert sum(int(x) for x in a[g16 == g]) > 1 << 64 and sum(int(x) for x in u[g16 == g]) > 1 << 64
    assert np.iinfo(np.int64).min in e and np.iinfo(np.int64).max in e
