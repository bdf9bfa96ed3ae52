"""Batch codes (batch_codes.cuh) against a plain value model: the tables tests/test_gpu_scan_codes_exact.py scans, and proof that
each of them holds what its case relies on.

A batch code numbers one distinct value of a dictionary-coded filter column for the whole page batch. Its key must be the value as
the per-block leaves compare it: a string's exact bytes; an integer's dictionary entry plus the block's base (sr.add), sign-fixed
when the block's record says so. So the tables put one value under many per-block layouts -- PAX dictionaries of different entry
widths, CS dictionaries with different bases and stream codecs, PAX and CS blocks of one column in one batch -- and reach the one
integer key that wraps (2^64 - 1: -1 of every signed type, the UINT64 maximum) and strings whose (length, 10-bit hash tag) collide.

The model is the generator's own cells: Python ints (unsigned types as unsigned), bytes, None for NULL. Checked here, without a
device: the oracle (oracle_binding.Block) decodes every cell of every table back to the model; a census of the bytes shows each
case is really there (entry widths per value, dictionary bases, -1 and the extremes, tag collisions, the mixed encodings of
OBGPU_ENC_AUTO columns, the const-ref and all-NULL CS blocks); the Python restatement of str_hash / key_of matches hand-computed
keys; and the model's distinct count per column. What the writer cannot produce is stated where the census meets it: a one-byte
type has one PAX entry width, and the PAX blocks of one type share one sign-fix state (the other state is that of the CS blocks
of the PAX + CS batch, which carry a base instead)."""
import functools

import numpy as np
import pytest

import oracle_binding as ora
from test_gpu_pipeline_exact import holds, leaf  # noqa: F401  (the row model's leaf and tree)
from test_gpu_scan_int_codes import TYPES, as_i64, bounds
from test_string_filter_exact import EDGE, header_facts

EQ, LE, LT, GE, GT, NE, BT, IN = range(8)          # OBGPU_WHITE_OP_*
RPB = 133
M64 = (1 << 64) - 1
OBJ_INT, OBJ_SMALLINT, OBJ_UINT64, OBJ_VARCHAR = 5, 2, 10, 22
ENC_RAW, ENC_DICT, ENC_RLE, ENC_CONST = 0, 1, 2, 3
ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STR_DICT, ENC_AUTO = 16, 17, 19, 32
CS_MODES = (1, 4, 6)                                # integer stream codecs: RAW, DELTA_ZIGZAG_RLE, SIMD_FIXEDPFOR
STR_LEN = 12                                        # the length every colliding string has
TYPE_IDS = [t[0] for t in TYPES]


class Table:
    """a table of the suite: the writer's image, the model cells per store column, each column's element width (0: string)"""

    def __init__(self, name, image, cells, widths, obj_types, proj=None):
        self.name, self.image, self.cells, self.widths, self.obj_types = name, image, cells, widths, obj_types
        self.proj = list(range(len(cells))) if proj is None else proj
        self.n = len(cells[0])
        self._sel = {}

    def selected(self, expr):
        k = repr(expr)
        if k not in self._sel:
            self._sel[k] = [r for r in range(self.n) if holds(expr, self.cells, r)]
        return self._sel[k]

    def distinct(self, col):
        return len({v for v in self.cells[col] if v is not None})


def cells_of(vals, nulls):
    return [None if z else v for v, z in zip(vals, nulls)]


def encode(cols, mode=1):
    """encode_table at RPB with CS integer stream codec `mode` (process-wide in the writer: RAW again after)"""
    import oceanbase_b200 as ob
    try:
        assert ob.capi.lib.obgpu_writer_set_cs_stream_encoding(mode) == 0
        return ob.encode_table(cols, RPB)
    finally:
        ob.capi.lib.obgpu_writer_set_cs_stream_encoding(1)


def elem_width(obj):
    return {19: 4, 21: 1}.get(obj, 8)


# ---- 1. integer layouts -----------------------------------------------------------------------------------------------------
KINDS = (0, 0, 0, 1, 2, 3, 0, 3, 1, 0, 2, 3, 0, 0, 1, 3)   # small, small, small, neg, mid, ext, ...: runs of small-value blocks
N_BLOCKS = len(KINDS)


def specials(bits, signed):
    """-1, 0, 1, the extremes and their neighbours (signed); 0, 1, the sign-bit neighbours and the extremes (unsigned)"""
    lo, hi = bounds(bits, signed)
    s = {lo, lo + 1, hi - 1, hi, 0, 1, 2}
    s |= {-1, -2} if signed else {hi >> 1, (hi >> 1) + 1}
    return sorted(s)


def block_pool(kind, bits, signed):
    """the values of a block of this kind: small magnitudes only (the narrowest entries), -1 / the top of an unsigned type next to
    small values, a middle width, the extremes"""
    lo, hi = bounds(bits, signed)
    if kind == 0:
        return [0, 1, 2, 3, 5, 7]
    if kind == 1:
        return [-1, -2, 0, 1, 2] if signed else [hi, hi - 1, 0, 1, 2]
    if kind == 2:
        return sorted({0, 1, 2, min(300, hi), min(70_000, hi)})
    return specials(bits, signed)


@functools.lru_cache(maxsize=None)
def int_layout_table(tname, byte_packing):
    import oceanbase_b200 as ob
    _, obj, bits, signed = next(t for t in TYPES if t[0] == tname)
    rng = np.random.default_rng(TYPE_IDS.index(tname) * 2 + byte_packing)
    vals, nulls = [], []
    for b, kind in enumerate(KINDS):
        pool = block_pool(kind, bits, signed)
        n = RPB if b + 1 < N_BLOCKS else RPB - 40          # a ragged last block
        blk = pool + [pool[int(k)] for k in rng.integers(0, len(pool), n - len(pool))]
        rng.shuffle(blk)
        vals += blk
        # NULLs only in every fourth block: the others can settle TRUE on the skip index
        nulls += (rng.random(n) < 0.1).tolist() if b % 4 == 1 else [False] * n
    n = len(vals)
    nz = np.array(nulls, dtype=np.uint8)
    cols = [ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64)),
            ob.Column(obj, ENC_DICT, as_i64(vals), nulls=nz, byte_packing_only=byte_packing)]
    t = Table("%s-%s" % (tname, "byte" if byte_packing else "bit"), ob.encode_table(cols, RPB), [list(range(n)), cells_of(vals, nulls)],
              [8, elem_width(obj)], [OBJ_INT, obj])
    t.cols = cols
    return t


def int_consts(bits, signed):
    lo, hi = bounds(bits, signed)
    return sorted({c for v in specials(bits, signed) for c in (v - 1, v, v + 1) if lo <= c <= hi})


def int_filters(ob, tname):
    """every range op at and around each special value; BT with equal, spanning and reversed bounds"""
    _, _, bits, signed = next(t for t in TYPES if t[0] == tname)
    lo, hi = bounds(bits, signed)
    W = ob.White
    out = [W(1, op, (c,)) for c in int_consts(bits, signed) for op in (EQ, NE, LT, LE, GT, GE)]
    for v in specials(bits, signed):
        out += [W(1, BT, (v, v)), W(1, BT, (lo, v)), W(1, BT, (v, hi))]
    out += [W(1, BT, (1, 0)), W(1, BT, (hi, lo))]
    return out


# ---- 2. CS dictionaries -----------------------------------------------------------------------------------------------------
CS_POOLS = ([0, 1, 2, 5, 9], [-1, 0, 1, 7], [-1000, -1, 0, 1, 300], [-(1 << 15), -1, 0, 1, (1 << 15) - 1])   # bases 0, -1, -1000, min
STRS = [b"", b"a", b"\x80", b"a\x80", b"a\x00", b"\x00", b"zz" * 7, b"apple", b"apples and pears"]


@functools.lru_cache(maxsize=None)
def cs_table(mode, pax=False):
    """0 row id; 1 INT, 2 SMALLINT, 3 UINT64 as CS_INT_DICT (PAX DICT when pax) with per-block bases; 4 VARCHAR CS_STR_DICT (PAX DICT)"""
    import oceanbase_b200 as ob
    rng = np.random.default_rng(50 + mode + 7 * pax)
    n = RPB * 12
    kinds = [(b // 2) % len(CS_POOLS) for b in range(12)]
    v1, v2, v3, s4 = [], [], [], []
    for k in kinds:
        pool = CS_POOLS[k]
        upool = [0, 1, 7] if k % 2 == 0 else [M64, M64 - 1, 1 << 63, (1 << 63) - 1, 1]
        for col, p in ((v1, pool), (v2, pool), (v3, upool), (s4, STRS[k:k + 5])):
            col += p + [p[int(j)] for j in rng.integers(0, len(p), RPB - len(p))]
    z = [(rng.random(n) < 0.08) for _ in range(4)]
    ie, se = (ENC_DICT, ENC_DICT) if pax else (ENC_CS_INT_DICT, ENC_CS_STR_DICT)
    cols = [ob.Column(OBJ_INT, ENC_RAW if pax else ENC_CS_INTEGER, np.arange(n, dtype=np.int64)),
            ob.Column(OBJ_INT, ie, as_i64(v1), nulls=z[0].astype(np.uint8)),
            ob.Column(OBJ_SMALLINT, ie, as_i64(v2), nulls=z[1].astype(np.uint8)),
            ob.Column(OBJ_UINT64, ie, as_i64(v3), nulls=z[2].astype(np.uint8)),
            ob.Column(OBJ_VARCHAR, se, s4, nulls=z[3].astype(np.uint8))]
    cells = [list(range(n)), cells_of(v1, z[0]), cells_of(v2, z[1]), cells_of(v3, z[2]), cells_of(s4, z[3])]
    t = Table("%s-%d" % ("pax" if pax else "cs", mode), encode(cols, mode), cells, [8, 8, 8, 8, 0],
              [OBJ_INT, OBJ_INT, OBJ_SMALLINT, OBJ_UINT64, OBJ_VARCHAR])
    t.cols = cols
    return t


@functools.lru_cache(maxsize=None)
def concat_table():
    """one batch of PAX blocks and CS blocks of the same columns"""
    import oceanbase_b200 as ob
    a, b = cs_table(1, pax=True), cs_table(4)
    img = ob.TableImage.concat([a.image, b.image])
    cells = [a.cells[c] + b.cells[c] for c in range(5)]     # each part keeps its own row ids in column 0
    return Table("pax+cs", img, cells, a.widths, a.obj_types)


@functools.lru_cache(maxsize=None)
def cs_uncodable_table():
    """0 row id; 1 CS_INT_DICT with one all-NULL block (a K_CONST plan); 2 CS_INT_DICT whose refs are const-encoded in every block
    (one value but 10 rows per block); 3 CS_INT_DICT that codes (so a scan still has a coded column next to them)"""
    import oceanbase_b200 as ob
    rng = np.random.default_rng(9)
    nb = 8
    n = RPB * nb
    v1 = [int(x) for x in rng.integers(-5, 5, n)]
    z1 = np.zeros(n, dtype=bool)
    z1[3 * RPB:4 * RPB] = True
    v2 = [42] * n
    for b in range(nb):
        for j in range(10):
            v2[b * RPB + 7 + 11 * j] = -1 - j
    v3 = [int(x) for x in rng.integers(-3, 40, n)]
    cols = [ob.Column(OBJ_INT, ENC_CS_INTEGER, np.arange(n, dtype=np.int64)),
            ob.Column(OBJ_INT, ENC_CS_INT_DICT, np.array(v1, dtype=np.int64), nulls=z1.astype(np.uint8)),
            ob.Column(OBJ_INT, ENC_CS_INT_DICT, np.array(v2, dtype=np.int64)),
            ob.Column(OBJ_INT, ENC_CS_INT_DICT, np.array(v3, dtype=np.int64))]
    return Table("cs-uncodable", encode(cols), [list(range(n)), cells_of(v1, z1), v2, v3], [8, 8, 8, 8], [OBJ_INT] * 4)


# ---- 3. strings -------------------------------------------------------------------------------------------------------------
G1, G2, MUL = 0x9E3779B97F4A7C15, 0xD6E8FEB86659FD93, 1 << 64


def str_hash(s):
    """bcodes::str_hash"""
    h = (G1 * (len(s) + 1)) % MUL
    for i in range(0, len(s), 8):
        h = ((h ^ int.from_bytes(s[i:i + 8], "little")) * G2) % MUL
        h ^= h >> 29
    h ^= h >> 32
    return (h * G1) % MUL


def key_of(abs_off, s):
    """bcodes::key_of: image offset (37 bits) | length (16) | hash tag (10) | 1"""
    return (abs_off << 27) | (len(s) << 11) | (((str_hash(s) >> 40) & 0x3FF) << 1) | 1


def tag_slot(strs):
    """(tag, home slot) of each string of STR_LEN bytes, vectorised over numpy uint64 (the same arithmetic as str_hash)"""
    a = np.frombuffer(b"".join(strs), dtype=np.uint8).reshape(-1, STR_LEN)
    w0 = np.ascontiguousarray(a[:, :8]).view("<u8")[:, 0]
    w1 = np.zeros(len(strs), dtype=np.uint64)
    for j in range(STR_LEN - 8):
        w1 |= a[:, 8 + j].astype(np.uint64) << np.uint64(8 * j)
    with np.errstate(over="ignore"):
        h = np.full(len(strs), (G1 * (STR_LEN + 1)) % MUL, dtype=np.uint64)
        for w in (w0, w1):
            h = (h ^ w) * np.uint64(G2)
            h ^= h >> np.uint64(29)
        h ^= h >> np.uint64(32)
        h = h * np.uint64(G1)
    return ((h >> np.uint64(40)) & np.uint64(0x3FF)).astype(np.int64), (h & np.uint64((1 << 18) - 1)).astype(np.int64)


@functools.lru_cache(maxsize=None)
def collision_pool():
    """several thousand distinct strings of STR_LEN bytes: pairs that share the tag and the home slot of the batch's table (a
    probe of one meets the other whatever the insertion order), the rest sharing tags by the pigeonhole"""
    cand = [b"\x80c%09d\xff" % i for i in range(1 << 18)]
    tag, slot = tag_slot(cand)
    key = tag * (1 << 18) + slot
    order = np.argsort(key, kind="stable")
    ks = key[order]
    same = np.flatnonzero(ks[1:] == ks[:-1])
    pairs = [(int(order[i]), int(order[i + 1])) for i in same[:40]]
    picked = [cand[i] for p in pairs for i in p]
    rest = [c for c in cand[:6000] if c not in set(picked)]
    return picked + rest[:4000 - len(picked)], len(pairs)


EXTRA = [b"", b"\x00", b"\x00" * 12, b"a\x00b", b"a\x80b", b"a\xffb", b"ab", b"a\x7fb", b"\xff" * 12, b"x" * 40]


@functools.lru_cache(maxsize=None)
def string_table():
    """0 row id; 1 VARCHAR DICT: the collision pool, with rows of other lengths in every block (a variable-length dictionary);
    2 VARCHAR DICT of EXTRA (empty, NUL bytes, strings that differ only in a byte >= 0x80); 3 INT RAW (no codes); 4 INT DICT"""
    import oceanbase_b200 as ob
    pool, _ = collision_pool()
    rng = np.random.default_rng(11)
    nb = len(pool) * 4 // (3 * RPB) + 2
    n = nb * RPB
    s1, k = [], 0
    for r in range(n):    # three rows in four from the pool; the fourth another length or NULL
        if r % 4 == 3:
            s1.append(EXTRA[(r // 4) % len(EXTRA)])
        else:
            s1.append(pool[k % len(pool)])
            k += 1
    s2 = [EXTRA[int(j)] for j in rng.integers(0, len(EXTRA), n)]
    v3 = [int(x) for x in rng.integers(-50, 50, n)]
    v4 = [int(x) for x in rng.integers(-3, 9, n)]
    z1, z2 = (np.arange(n) % 4 == 3) & (rng.random(n) < 0.3), rng.random(n) < 0.1
    cols = [ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(OBJ_VARCHAR, ENC_DICT, s1, nulls=z1.astype(np.uint8)),
            ob.Column(OBJ_VARCHAR, ENC_DICT, s2, nulls=z2.astype(np.uint8)), ob.Column(OBJ_INT, ENC_RAW, np.array(v3, dtype=np.int64)),
            ob.Column(OBJ_INT, ENC_DICT, np.array(v4, dtype=np.int64))]
    return Table("strings", ob.encode_table(cols, RPB), [list(range(n)), cells_of(s1, z1), cells_of(s2, z2), v3, v4], [8, 0, 0, 8, 8],
                 [OBJ_INT, OBJ_VARCHAR, OBJ_VARCHAR, OBJ_INT, OBJ_INT])


# ---- 4. mixed encodings -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def auto_table():
    """OBGPU_ENC_AUTO columns whose blocks differ in shape: one value (CONST), long runs (RLE), few values (DICT), all distinct
    (RAW): 1 INT, 2 VARCHAR; 3 an INT DICT column that codes"""
    import oceanbase_b200 as ob
    rng = np.random.default_rng(13)
    nb = 12
    v1, s2 = [], []
    for b in range(nb):
        shape = b % 4
        if shape == 0:
            blk = [-1] * RPB
        elif shape == 1:
            blk = [int(x) for x in np.repeat(rng.integers(-9, 9, 3), 45)[:RPB]]
        elif shape == 2:
            blk = [int(x) for x in rng.choice([-1, 0, 1, 1 << 40, -(1 << 50)], RPB)]
        else:
            blk = [int(x) for x in rng.integers(-(1 << 62), 1 << 62, RPB)]
        v1 += blk
        s2 += [b"s%d" % (v % 1000) if shape < 3 else b"u%dx%d" % (b, j) for j, v in enumerate(blk)]
    n = nb * RPB
    v3 = [int(x) for x in rng.integers(0, 20, n)]
    cols = [ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(OBJ_INT, ENC_AUTO, np.array(v1, dtype=np.int64)),
            ob.Column(OBJ_VARCHAR, ENC_AUTO, s2), ob.Column(OBJ_INT, ENC_DICT, np.array(v3, dtype=np.int64))]
    return Table("auto", ob.encode_table(cols, RPB), [list(range(n)), v1, s2, v3], [8, 8, 0, 8], [OBJ_INT, OBJ_INT, OBJ_VARCHAR, OBJ_INT])


# ---- 5. the code cap --------------------------------------------------------------------------------------------------------
CAP = 65536


@functools.lru_cache(maxsize=None)
def cap_table():
    """1: exactly 65 536 distinct INT values (the most that is coded); 2: 65 537 (the fewest over the cap); spread over the
    blocks so that every block holds a few hundred different values in a sorted DICT"""
    import oceanbase_b200 as ob
    n = CAP + 1 + 3 * RPB
    perm = np.random.default_rng(17).permutation(n)
    v2 = np.where(perm <= CAP, perm, perm % 100) * 7 - 200_000             # values 0..65536 (times 7): 65 537 distinct
    v1 = np.where(perm < CAP, perm, perm % 100) * 5 - 100_000              # values 0..65535 (times 5): 65 536 distinct
    cols = [ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(OBJ_INT, ENC_DICT, v1.astype(np.int64)),
            ob.Column(OBJ_INT, ENC_DICT, v2.astype(np.int64))]
    return Table("cap", ob.encode_table(cols, RPB), [list(range(n)), v1.tolist(), v2.tolist()], [8, 8, 8], [OBJ_INT] * 3)


# ---- 7. open paths ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def open_table():
    """the INT layout table with a string column: 0 row id, 1 INT DICT (every layout), 2 VARCHAR DICT, 3 UINT64 DICT"""
    import oceanbase_b200 as ob
    a, u = int_layout_table("int", False), int_layout_table("uint64", True)
    n = a.n
    rng = np.random.default_rng(19)
    s2 = [EXTRA[int(j)] for j in rng.integers(0, len(EXTRA), n)]
    cols = [a.cols[0], a.cols[1], ob.Column(OBJ_VARCHAR, ENC_DICT, s2), u.cols[1]]
    return Table("open", ob.encode_table(cols, RPB), [a.cells[0], a.cells[1], s2, u.cells[1]], [8, 8, 0, 8],
                 [OBJ_INT, OBJ_INT, OBJ_VARCHAR, OBJ_UINT64])


# ---- 8. the bench shape -----------------------------------------------------------------------------------------------------
BENCH_ROWS, BENCH_SEED = 300_000, 3


@functools.lru_cache(maxsize=None)
def bench_rpb():
    from oceanbase_b200.synth import make_config3_like, rows_per_block_for_target
    return rows_per_block_for_target(make_config3_like, seed=BENCH_SEED)


@functools.lru_cache(maxsize=None)
def bench_workload():
    from oceanbase_b200.synth import make_config3_like
    return make_config3_like(rows=BENCH_ROWS, rows_per_block=bench_rpb(), seed=BENCH_SEED)


@functools.lru_cache(maxsize=None)
def bench_model():
    """the cfg3 columns rebuilt from the generator's seeds in numpy: ints as int64 arrays, strings as (heap, offsets, rank)"""
    from oceanbase_b200.synth import _col_seed, _string_dict, _zipf_ranks, splitmix64
    s = lambda c: _col_seed(BENCH_SEED, c)
    ints = {}
    for c, card in enumerate([16, 64, 256, 4096, 16, 1024, 65536, 200]):
        vals = (splitmix64(s(c) + 5, 0, card) >> np.uint64(20)).astype(np.int64)
        if c == 3:
            vals = np.arange(card, dtype=np.int64) * 1000
        ints[c] = (vals, _zipf_ranks(s(c), 0, BENCH_ROWS, card))
    strs = {c: (_string_dict(s(c) + 3, 1024), _zipf_ranks(s(c), 0, BENCH_ROWS, 1024)) for c in range(8, 16)}
    return ints, strs


def bench_string(strs, c, k):
    (heap, off), _ = strs[c]
    return bytes(heap[off[k]:off[k + 1]])


# ---- the census helpers ------------------------------------------------------------------------------------------------------
def pax_dict_width(table, b, col):
    """ObDictMetaHeader::data_size_ of a PAX DICT column in block b (the dictionary's entry width)"""
    img, o = np.asarray(table.image), int(table.offsets[b])
    hs = int(img[o + 4:o + 8].view(np.uint32)[0])
    n_cols = int(img[o + 10:o + 12].view(np.uint16)[0])
    h = img[o + hs + 16 * col:o + hs + 16 * col + 16]
    dm = o + hs + 16 * n_cols + int(h[8:12].view(np.uint32)[0])
    return int(img[dm + 6:dm + 8].view(np.uint16)[0])


def block_dicts(table, col):
    """per block: the dictionary entries the oracle reads (ints as their 64-bit image)"""
    out = []
    for b in range(table.n_blocks):
        blk = ora.Block(table.block(b))
        out.append([blk.dict_entry(col, e)[0] for e in range(blk.dict_count(col))])
    ora.arena_reset()
    return out


def decode_all(t, image=None):
    """every cell of every block through the oracle, against the model"""
    image = t.image if image is None else image
    r0 = 0
    for b in range(image.n_blocks):
        blk = ora.Block(image.block(b))
        for c in range(len(t.cells)):
            got = [blk.cell(c, r) for r in range(blk.row_count)]
            want = t.cells[c][r0:r0 + blk.row_count]
            if t.widths[c]:   # the oracle gives an integer's image at its datum length
                mask = (1 << 8 * t.widths[c]) - 1
                want = [None if v is None else v & mask for v in want]
                got = [None if v is None else v & mask for v in got]
            assert got == want, (t.name, b, c)
        r0 += blk.row_count
        ora.arena_reset()
    assert r0 == t.n


# ---- the tests ----------------------------------------------------------------------------------------------------------------
def test_str_hash_restatement_matches_hand_computed_keys():
    # the empty string: h = G1 * 1, h ^= h >> 32, h *= G1 (no 8-byte step)
    h = G1 ^ (G1 >> 32)
    assert str_hash(b"") == (h * G1) % MUL
    # one step of "a" (0x61), worked by hand in the same order as the device loop
    h = ((((G1 * 2) % MUL) ^ 0x61) * G2) % MUL
    h ^= h >> 29
    h ^= h >> 32
    assert str_hash(b"a") == (h * G1) % MUL
    assert key_of(0, b"") == 1 | (((str_hash(b"") >> 40) & 0x3FF) << 1)
    assert key_of(5, b"abc") >> 27 == 5 and (key_of(5, b"abc") >> 11) & 0xFFFF == 3
    # the vectorised form used for the search agrees with the scalar one
    probe = [b"\x80c%09d\xff" % i for i in (0, 1, 77, 123456)]
    tags, slots = tag_slot(probe)
    for s, t, sl in zip(probe, tags, slots):
        assert (str_hash(s) >> 40) & 0x3FF == t and str_hash(s) & ((1 << 18) - 1) == sl


@pytest.mark.parametrize("tname", TYPE_IDS)
@pytest.mark.parametrize("byte_packing", [True, False], ids=["byte_refs", "bit_refs"])
def test_int_layout_tables(tname, byte_packing):
    t = int_layout_table(tname, byte_packing)
    decode_all(t)
    _, obj, bits, signed = next(x for x in TYPES if x[0] == tname)
    lo, hi = bounds(bits, signed)
    assert {int(h[0]) for h in header_facts(t.image, 1)} == {ENC_DICT}
    # census: the specials are stored, and one value is stored under different entry widths where the type allows it
    present = {v for v in t.cells[1] if v is not None}
    assert set(specials(bits, signed)) <= present
    widths = {}
    for b in range(t.image.n_blocks):
        w = pax_dict_width(t.image, b, 1)
        for v in {x for x in t.cells[1][b * RPB:(b + 1) * RPB] if x is not None}:
            widths.setdefault(v, set()).add(w)
    multi = {v for v, ws in widths.items() if len(ws) > 1}
    if bits > 8:
        assert {0, 1, 2} <= multi, (tname, {v: widths[v] for v in (0, 1, 2)})
    else:   # a one-byte type has one entry width: every value keeps its layout
        assert not multi
    # the value whose integer key wraps (2^64 - 1 after the sign fix) is stored in every signed type and in UINT64
    if signed or bits == 64:
        assert (-1 if signed else M64) in present
    assert t.distinct(1) == len(present)


@pytest.mark.parametrize("mode", CS_MODES)
def test_cs_tables(mode):
    t = cs_table(mode)
    decode_all(t, ora.cs_transform_table(t.image) if mode != 1 else None)
    pax = cs_table(1, pax=True)
    decode_all(pax)
    assert {int(h[0]) for h in header_facts(t.image, 1)} == {2} and {int(h[0]) for h in header_facts(t.image, 4)} == {3}
    # census: blocks whose dictionaries start at different minima -- the writer's base is a block's minimum when it is negative --
    # hold one common value (-1 and 0); PAX blocks of the same columns keep base 0
    img = ora.cs_transform_table(t.image) if mode != 1 else t.image
    for col in (1, 2):
        dicts = block_dicts(img, col)
        bases = {min(d) if min(d) < 0 else 0 for d in (sign64(x) for x in dicts) if d}
        assert len(bases) >= 3, bases
        with_m1 = [d for d in (sign64(x) for x in dicts) if -1 in d]
        assert len({min(d) for d in with_m1}) >= 2
    assert all(-1 in t.cells[c] and 0 in t.cells[c] for c in (1, 2)) and M64 in t.cells[3]


def sign64(xs):
    return [x - (1 << 64) if x >= 1 << 63 else x for x in xs]


def test_concat_and_uncodable_cs_tables():
    t = concat_table()
    a, b = cs_table(1, pax=True), cs_table(4)
    assert t.image.n_blocks == a.image.n_blocks + b.image.n_blocks and t.n == a.n + b.n
    assert [int(h[0]) for h in header_facts(t.image, 1)] == [ENC_DICT] * a.image.n_blocks + [2] * b.image.n_blocks
    decode_all(a)
    u = cs_uncodable_table()
    decode_all(u)
    # census: one block of column 1 is all NULL (no dictionary); column 2 meets the writer's const-ref rule in every block (one
    # ref covers all but <= 64 rows and fewer than 10 % of the block)
    counts = [ora.Block(u.image.block(b)).dict_count(1) for b in range(u.image.n_blocks)]
    assert counts.count(0) == 1
    for b in range(u.image.n_blocks):
        cells = u.cells[2][b * RPB:(b + 1) * RPB]
        exc = len(cells) - max(cells.count(v) for v in set(cells))
        assert 0 < exc <= 64 and exc < len(cells) * 10 // 100
    ora.arena_reset()


def test_string_table():
    t = string_table()
    decode_all(t)
    pool, n_pairs = collision_pool()
    assert len(pool) >= 3000 and len(set(pool)) == len(pool) and {len(s) for s in pool} == {STR_LEN}
    # census: pairs with one (length, tag) and one home slot, and tags shared by many more strings of the length
    tags, slots = tag_slot(pool)
    assert n_pairs >= 10
    assert len(set(zip(tags.tolist(), slots.tolist()))) <= len(pool) - n_pairs
    assert len(set(tags.tolist())) <= 1024 < len(pool)
    present = {v for v in t.cells[1] if v is not None}
    assert set(pool) <= present
    # every block's dictionary has entries of more than one length: a variable-length dictionary (what stage records take)
    for b in range(t.image.n_blocks):
        assert len({len(s) for s in t.cells[1][b * RPB:(b + 1) * RPB] if s is not None}) > 1, b
    assert {b"", b"a\x80b", b"a\xffb", b"\x00" * 12} <= set(t.cells[2])
    assert t.distinct(1) == len(present)


def test_auto_table_mixes_encodings():
    t = auto_table()
    decode_all(t)
    for col in (1, 2):
        kinds = {int(h[0]) for h in header_facts(t.image, col)}
        assert ENC_DICT in kinds and kinds - {ENC_DICT}, (col, kinds)


def test_cap_table():
    t = cap_table()
    assert t.distinct(1) == CAP and t.distinct(2) == CAP + 1
    decode_all(t)
    assert {int(h[0]) for h in header_facts(t.image, 1)} == {ENC_DICT} == {int(h[0]) for h in header_facts(t.image, 2)}


def test_open_table():
    t = open_table()
    decode_all(t)
    assert -1 in t.cells[1] and M64 in t.cells[3]


def test_bench_segment_matches_its_seeds():
    """the bench's table at its own block cut, decoded: every cell equals the numpy rebuild of its seeds"""
    w = bench_workload()
    assert 100 <= w.rows_per_block <= 200 and w.table.total_rows == BENCH_ROWS
    ints, strs = bench_model()
    r0 = 0
    for b in range(0, w.table.n_blocks, 37):
        blk = ora.Block(w.table.block(b))
        r0 = b * w.rows_per_block
        for c in (0, 1, 3, 6):
            vals, ranks = ints[c]
            assert [blk.cell(c, r) for r in range(blk.row_count)] == vals[ranks[r0:r0 + blk.row_count]].tolist(), (b, c)
        for c in (8, 9, 10):
            ranks = strs[c][1]
            assert [blk.cell(c, r) for r in range(blk.row_count)] == [bench_string(strs, c, int(k)) for k in ranks[r0:r0 + blk.row_count]]
        ora.arena_reset()
