"""CS integer streams under every stream codec, checked against the values that were written (the device half is
tests/test_gpu_cs_stream_exact.py).

A CS block (CS_ENCODING_ROW_STORE) may store each integer stream -- CS_INTEGER values, CS_INT_DICT values and refs, CS_STRING
END offsets, CS_STR_DICT offsets and refs -- with DOUBLE_DELTA_ZIGZAG_RLE (2), DOUBLE_DELTA_ZIGZAG_PFOR (3), DELTA_ZIGZAG_RLE (4),
DELTA_ZIGZAG_PFOR (5), SIMD_FIXEDPFOR (6) or XOR_FIXED_PFOR (8). A batch opened on the device restates every such block as RAW
(stream_codecs.cuh) and every later kernel reads only that restatement, so a decoder slip is a silently wrong value.

1. Stream matrix: the oracle KAT's streams (test_stream_codec_kat.datasets: every shape, width and length), plus runs separated by
   jumps of +-2^k (every RLE escape length, the high-part-first split of 8-byte deltas wider than 45 bits), 20..300 equal deltas in
   a row (RLE repeat records, counts of one and two bytes) and sparse top-bit spikes (PFOR exceptions of the full width), each
   written as one UINT64 CS_INTEGER column without NULLs, one single-block table per length, under every codec mode. A census
   walks the coded streams and fails when a path the decoders have is not reached: per codec and stored width a coded stream,
   a tail-only stream (< 128 values), the PFOR exception flag in the first block, and every RLE code kind (1-bit zero, N2 / N3 /
   N4 tiers, each escape length the encoder emits at that width, repeat records).
2. Column matrix: CS_INTEGER columns of every integer type at 0 / 10 / 100 % NULL, shaped to reach each way the writer stores a
   block (plain, base, NULL replaced by nmax + 1 or nmin - 1, NULL bitmap: the form asserted per block against a restatement
   of the writer's rule), CS_INT_DICT, CS_STRING (empty strings, END offsets of one, two and four bytes) and CS_STR_DICT columns.
3. Block sizes of 1, 127, 128, 129 and 2051 rows; a block whose restatement needs four-byte END offsets although its coded form
   is far smaller, and one that crosses from one- to two-byte END offsets.

CPU checks: the oracle's restatement (ora.cs_transform) equals the RAW-written twin byte for byte and decodes every cell back
to the written value; its filters select exactly the model's rows."""
import functools

import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import TYPES, _draw, as_store, datum_len, oracle_value
from test_cs_stream_codecs import MODES, stream_types
from test_stream_codec_kat import WIDTHS, datasets

CODECS = (2, 3, 4, 5, 6, 8)
RLE = (2, 4)
PFOR = (3, 5, 6, 8)
OBJ_INT, OBJ_UINT64, OBJ_VARCHAR = 5, 10, 22
ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STRING, ENC_CS_STR_DICT = 16, 17, 18, 19
HEADER_TYPE = {ENC_CS_INTEGER: 0, ENC_CS_STRING: 1, ENC_CS_INT_DICT: 2, ENC_CS_STR_DICT: 3}
BT, NU, EQ = 6, 8, 0                                            # OBGPU_WHITE_OP_*
# RLE bit tiers N2 / N3 / N4 per stored width (ob_bp_util.h); a zigzag delta at or above 2^(N4 - 1) takes an escape of
# (its byte length) bytes, so widths 1 and 2 have no escapes and width 4 only 3- and 4-byte ones
RLE_TIERS = {1: (3, 5, 9), 2: (6, 12, 17), 4: (6, 10, 17), 8: (6, 12, 20)}
ESCAPES = {1: set(), 2: set(), 4: {3, 4}, 8: {3, 4, 5, 6, 7, 8}}
STORE_SIZE = {1: 1, 2: 2, 3: 4, 4: 4, 5: 8, 6: 1, 7: 2, 8: 4, 9: 4, 10: 8, 19: 4, 21: 1}   # type_store_size (ob_format.h)
SIGNED = {1, 2, 3, 4, 5, 19}


def encode_with(mode, cols, rpb):
    """encode_table with integer stream codec `mode` (obgpu_writer_set_cs_stream_encoding is process-wide: RAW again after)"""
    import oceanbase_b200 as ob
    lib = ob.capi.lib
    try:
        assert lib.obgpu_writer_set_cs_stream_encoding(mode) == 0
        return ob.encode_table(cols, rpb)
    finally:
        lib.obgpu_writer_set_cs_stream_encoding(1)


# ---- 1. the stream matrix ------------------------------------------------------------------------------------------------
def extra_shapes(dt, n):
    """the shapes the KAT lacks, as (name, array) of length n"""
    bits = np.dtype(dt).itemsize * 8
    top = (1 << bits) - 1
    rng = np.random.default_rng(bits)
    # runs of equal values separated by jumps of +-2^k, k = 1 .. bits - 1
    jumps = [s << k for k in range(1, bits) for s in (1, -1)]
    v, out = (1 << (bits - 1)) + 12345, []
    while len(out) < n:
        for j in jumps:
            out += [v & top] * int(rng.integers(1, 30))
            v += j
    jumps_a = np.array(out[:n], dtype=np.uint64).astype(dt)
    # 20..300 equal deltas in a row (a zero delta among them)
    out, v = [], 7
    while len(out) < n:
        d = [0, 1, 3, -2, 1000, int(rng.integers(0, top, dtype=np.uint64, endpoint=True))][len(out) % 6]
        for _ in range(int(rng.integers(20, 301))):
            out.append(v & top)
            v += d
    ramps = np.array(out[:n], dtype=np.uint64).astype(dt)
    # zeros with sparse spikes of the top and the lowest bit: every PFOR codec takes exceptions of the full width (bx = bits)
    sparse = np.zeros(n, dtype=np.uint64)
    sparse[7::50] = (1 << (bits - 1)) | 1
    return [("jumps", jumps_a), ("ramps", ramps), ("sparse_top", sparse.astype(dt))]


def stream_shapes(ub):
    """{length: [(shape name, array)]}: the KAT's datasets at width ub plus extra_shapes, grouped by length"""
    dt = WIDTHS[ub]
    by_n = {}
    for name, a in datasets(dt, np.random.default_rng(500 + ub)):
        by_n.setdefault(a.size, []).append((name, a))
    for n, shapes in by_n.items():
        shapes += extra_shapes(dt, n)
    return by_n


def uint64_cols(shapes):
    import oceanbase_b200 as ob
    return [ob.Column(OBJ_UINT64, ENC_CS_INTEGER, np.ascontiguousarray(a.astype(np.uint64)).view(np.int64)) for _, a in shapes]


@functools.lru_cache(maxsize=None)
def stream_matrix(mode, ub):
    """(coded table, RAW twin, values[block][column] as uint64): one single-block table per length, concatenated"""
    from oceanbase_b200.sstable import TableImage
    coded, raw, values = [], [], []
    for n, shapes in sorted(stream_shapes(ub).items()):
        coded.append(encode_with(mode, uint64_cols(shapes), n))
        raw.append(encode_with(1, uint64_cols(shapes), n))
        values.append([a.astype(np.uint64) for _, a in shapes])
    return TableImage.concat(coded), TableImage.concat(raw), values


def stream_layout(block):
    """Every stream of a CS block, in stream order: (column, ObIntegerStream::EncodingType (None for a string stream), width tag
    (byte 3 of the stream meta), block offset of the stream, block offset of its END, value count). The walk of stream_types,
    which gives the types only; the two must agree."""
    hs = int(block[4:8].view(np.uint32)[0])
    ncol = int(block[10:12].view(np.uint16)[0])
    rows = int(block[16:20].view(np.uint32)[0])
    ah = block[hs:hs + 12]
    offsets_len, n_streams = int(ah[6:10].view(np.uint32)[0]), int(ah[10:12].view(np.uint16)[0])
    so = block[len(block) - offsets_len:]
    ow = 1 << int(so[3])
    ends = so[5:5 + ow * n_streams].view({1: np.uint8, 2: np.uint16, 4: np.uint32}[ow]).astype(np.int64)
    pos, si, out = hs + 12 + 4 * ncol, 0, []
    bmb = (rows + 7) // 8
    for c in range(ncol):
        t, attrs = int(block[hs + 12 + 4 * c + 1]), int(block[hs + 12 + 4 * c + 2])
        if t in (0, 1):
            meta = (bmb if attrs & 2 else 0) + (bmb if attrs & 8 else 0)
            kinds = [False] if t == 0 else ([True] if attrs & 1 else [True, False])
            counts = [rows, rows]
        else:
            meta = 10 + (bmb if attrs & 8 else 0)
            distinct = int(block[pos + 2:pos + 6].view(np.uint32)[0])
            refs = int(block[pos + 6:pos + 10].view(np.uint32)[0]) if block[pos + 1] & 4 else rows
            kinds = [] if distinct == 0 else ([False, False] if t == 2 else ([True, False] if attrs & 1 else [True, False, False]))
            counts = [distinct, refs] if t == 2 else ([0, refs] if attrs & 1 else [0, distinct, refs])
        at = pos + meta
        for is_str, cnt in zip(kinds, counts):
            t_w = (None, None) if is_str else (int(block[at + 2]), int(block[at + 3]))
            out.append((c,) + t_w + (at, int(ends[si]), cnt))
            at = int(ends[si])
            si += 1
        pos = pos + meta if not kinds else at
    assert [s[1] for s in out] == stream_types(block)
    return out


def stream_meta(block, at):
    """(meta length, base or None, NULL replacement or None) of the ObIntegerStreamMeta at `at`"""
    version, attr, pos, vals = int(block[at]), int(block[at + 1]), at + 4, []
    for k in range(2):
        if not attr & (1 << k):
            vals.append(None)
            continue
        v, sh = 0, 0
        while True:
            b = int(block[pos])
            pos += 1
            v |= (b & 0x7F) << sh
            sh += 7
            if not b & 0x80:
                break
        vals.append(v)
    return pos + (1 if version > 0 else 0) - at, vals[0], vals[1]


def coded_streams(block):
    """(codec, stored width, codec bytes, value count) of every non-RAW integer stream of a block"""
    out = []
    for _, t, wtag, at, end, cnt in stream_layout(block):
        if t in (None, 1):
            continue
        ml = stream_meta(block, at)[0]
        out.append((t, 1 << wtag, bytes(block[at + ml:end]), cnt))
    return out


def pfor_facts(p, wb, count, xor):
    """what one PFOR-family stream holds, block by block: [xb (XOR)][b | 0x80 with exceptions]([bx][bitmap 16 B]
    [exceptions, xn x bx bits])[n x b bits]"""
    facts, pos, done = set(), 0, 0
    while done < count:
        n = min(128, count - done)
        if xor:
            facts.add("xb_all" if p[pos] >= wb * 8 else ("xb" if p[pos] else "xb0"))
            pos += 1
        b = p[pos]
        pos += 1
        if n == 128 and b & 0x80:
            b &= 0x7F
            bx, xm = p[pos], int.from_bytes(p[pos + 1:pos + 17], "little")
            pos += 17
            xn = bin(xm).count("1")
            facts.add("exc_first" if done == 0 else "exc")
            if xm & ((1 << 64) - 1) and xm >> 64:
                facts.add("exc_both_halves")
            if xn * bx % 8:
                facts.add("exc_partial_byte")
            if bx == 64:
                facts.add("bx64")
            pos += (xn * bx + 7) // 8
        if b == 64:
            facts.add("b64")
        pos += (n * b + 7) // 8
        done += n
    assert pos == len(p), (pos, len(p))
    return facts


def rle_facts(p, wb, count):
    """the code kinds of one RLE-family stream (LSB-first): 1 zero delta | 01 N2 | 001 N3 | 0001 N4 | 0000 + 3 bits k: k = 0
    repeat record (3 bits bytes - 1, then that many bytes of count - 18), else an escape of k + 1 bytes. Prefixes are read and
    payloads skipped; only repeat counts are read, to know where the stream ends."""
    n2, n3, n4 = RLE_TIERS[wb]
    pad = p + bytes(16)

    def get(bit, w):
        return (int.from_bytes(pad[bit >> 3:(bit >> 3) + 10], "little") >> (bit & 7)) & ((1 << w) - 1)

    facts, bit, done = set(), 0, 0
    while done < count:
        if get(bit, 1):
            facts.add("zero")
            bit += 1
        elif get(bit + 1, 1):
            facts.add("n2")
            bit += 2 + n2
        elif get(bit + 2, 1):
            facts.add("n3")
            bit += 3 + n3
        elif get(bit + 3, 1):
            facts.add("n4")
            bit += 4 + n4
        else:
            k = get(bit + 4, 3)
            bit += 7
            if k == 0:
                nb = get(bit, 3) + 1
                done += get(bit + 3, 8 * nb) + 18
                facts.add(("repeat", nb))
                bit += 3 + 8 * nb
                continue
            facts.add(("escape", k + 1))
            bit += 8 * (k + 1)
        done += 1
    assert done == count and (bit + 7) // 8 == len(p), (done, count, bit, len(p))
    return facts


def stream_facts(t, wb, p, count):
    facts = {"stored"} | ({"tail_only"} if count < 128 else set())
    if t in RLE:
        return facts | rle_facts(p, wb, count)
    return facts | pfor_facts(p, wb, count, xor=t == 8)


@functools.lru_cache(maxsize=None)
def census():
    """{(codec, stored width): facts seen} over the stream matrix of every forced codec"""
    seen = {}
    for mode in CODECS:
        for ub in WIDTHS:
            table = stream_matrix(mode, ub)[0]
            for i in range(table.n_blocks):
                for t, wb, p, cnt in coded_streams(table.block(i)):
                    assert t == mode
                    seen.setdefault((t, wb), set()).update(stream_facts(t, wb, p, cnt))
    return seen


def test_census_reaches_every_decoder_path():
    seen = census()
    for t in CODECS:
        for wb in WIDTHS:
            f = seen.get((t, wb), set())
            assert {"stored", "tail_only"} <= f, (MODES[t], wb, f)
            if t in PFOR:
                assert "exc_first" in f, (MODES[t], wb)
            if t in RLE:
                assert {"zero", "n2", "n3", "n4", ("repeat", 1), ("repeat", 2)} <= f, (MODES[t], wb, f)
                assert {k for kind, k in (x for x in f if isinstance(x, tuple)) if kind == "escape"} == ESCAPES[wb], (MODES[t], wb, f)
        if t in PFOR:
            # exception bitmaps with rows on both sides of row 64, exception payloads ending inside a byte, and b / bx of 64
            assert any("exc_both_halves" in seen[(t, wb)] for wb in WIDTHS), MODES[t]
            assert any("exc_partial_byte" in seen[(t, wb)] for wb in WIDTHS), MODES[t]
            assert {"b64", "bx64"} <= seen[(t, 8)], (MODES[t], seen[(t, 8)])
    for wb in WIDTHS:       # XOR's per-block shift: none, part of the width, the whole width (a block of equal values)
        assert {"xb0", "xb", "xb_all"} <= seen[(8, wb)], (wb, seen[(8, wb)])


@pytest.mark.parametrize("ub", sorted(WIDTHS))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_stream_matrix_restates_to_the_raw_twin(mode, ub):
    table, raw, values = stream_matrix(mode, ub)
    assert table.n_blocks == raw.n_blocks == len(values)
    coded = 0
    for i in range(table.n_blocks):
        blk, twin = table.block(i), raw.block(i)
        hs = int(blk[4:8].view(np.uint32)[0])
        coded += len(coded_streams(blk))
        t = ora.cs_transform(blk)
        assert t.size == twin.size and np.array_equal(t[hs:], twin[hs:]), (MODES[mode], ub, i)
        b = ora.Block(t)
        rid = np.arange(b.row_count, dtype=np.int32)
        for c, want in enumerate(values[i]):
            d, nulls, _ = b.get_rows_fixed(c, rid)
            assert not nulls.any() and np.array_equal(d.view(np.uint64)[:len(want)], want), (MODES[mode], ub, i, c)
    assert coded > 0, MODES[mode]


# ---- 2. the column matrix --------------------------------------------------------------------------------------------------
SIGNED_T = ("tinyint", "smallint", "mediumint", "int32", "int", "date")
UNSIGNED_T = ("utinyint", "usmallint", "umediumint", "uint32", "uint64", "year")
INT_SHAPES = ("ext", "spike", "mono", "zero_top", "small", "mid")
NULL_RATES = {"n0": 0.0, "n10": 0.10, "n100": 1.0}
GROUPS = ("signed", "unsigned", "dict_str")
# (mode, rows per block): every codec mode at 129 rows per block, some at 1, 127, 128 and 2051
COLUMN_TABLES = [(m, 129) for m in sorted(MODES)] + [(6, 1), (0, 2051), (2, 127), (3, 128), (4, 2051), (5, 1), (8, 128)]
ROWS = {1: 64, 127: 600, 128: 600, 129: 600, 2051: 4300}


def int_shape(rng, tname, shape, n):
    """n values of the type: 'ext' type extremes, 0 and -1 among draws over the whole range (the minimum and the maximum every
    60 rows); 'spike' a small band above lo / 2 (signed) or 100 with 5 % spikes to the maximum; 'mono' sorted draws strictly inside
    the range; 'zero_top' 0 and the maximum every 50 rows among non-negative draws; 'small' / 'mid' values within +-60 / +-20000
    (signed) or 0..120 / 0..40000 (unsigned)"""
    _, lo, hi = TYPES[tname]
    if shape == "ext":
        sp = [lo, hi, 0] + ([-1] if lo < 0 else [])
        v = [sp[int(rng.integers(0, len(sp)))] if rng.random() < 0.35 else x for x in _draw(rng, lo, hi, n)]
        v[1::60] = [lo] * len(v[1::60])
        v[2::60] = [hi] * len(v[2::60])
        return v
    if shape == "spike":
        b0 = lo // 2 if lo < 0 else 100
        return [hi if s else b0 + int(x) for x, s in zip(rng.integers(0, 16, size=n), rng.random(n) < 0.05)]
    if shape == "mono":
        return sorted(_draw(rng, lo + 1, hi - 1, n))
    if shape == "zero_top":
        v = _draw(rng, 0, hi, n)
        v[3::50] = [0] * len(v[3::50])
        v[4::50] = [hi] * len(v[4::50])
        return v
    span = 60 if shape == "small" else 20000
    return _draw(rng, max(lo, -span), min(hi, span), n) if lo < 0 else _draw(rng, 0, min(hi, 2 * span), n)


def null_mask(rng, rate, n):
    return (rng.random(n) < rate).astype(np.uint8) if rate < 1.0 else np.ones(n, dtype=np.uint8)


class Spec:
    """One column-matrix table: the writer's columns, the true value (int, bytes or None) of every cell, and per column its
    ObObjType, encoding and name"""

    def __init__(self, cols, truth, names):
        self.cols, self.truth, self.names = cols, truth, names
        self.obj = [c.obj_type for c in cols]
        self.enc = [c.encoding for c in cols]
        self.n = len(truth[0])

    def is_str(self, c):
        return self.obj[c] == OBJ_VARCHAR


def with_nulls(values, mask):
    return [None if m else v for v, m in zip(values, mask.tolist())]


def strings(rng, n, lo, hi, pool=None):
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz\x00\x80\xff", dtype=np.uint8)
    if pool is not None:
        return [pool[int(i)] for i in rng.integers(0, len(pool), size=n)]
    return [bytes(alpha[rng.integers(0, len(alpha), size=int(k))]) for k in rng.integers(lo, hi + 1, size=n)]


@functools.lru_cache(maxsize=None)
def column_spec(group, n):
    import oceanbase_b200 as ob
    rng = np.random.default_rng(7000 + GROUPS.index(group) * 100 + n)
    cols, truth, names = [], [], []

    def add(obj, enc, values, rate, name):
        m = null_mask(rng, rate, len(values))
        if enc in (ENC_CS_STRING, ENC_CS_STR_DICT):
            cols.append(ob.Column(obj, enc, values, nulls=m))
        else:
            cols.append(ob.Column(obj, enc, as_store(values), nulls=m))
        truth.append(with_nulls(values, m))
        names.append(name)

    if group != "dict_str":
        for tname in (SIGNED_T if group == "signed" else UNSIGNED_T):
            obj = TYPES[tname][0]
            for shape in INT_SHAPES:
                for nname in ("n0", "n10"):
                    add(obj, ENC_CS_INTEGER, int_shape(rng, tname, shape, n), NULL_RATES[nname], (tname, shape, nname))
            add(obj, ENC_CS_INTEGER, int_shape(rng, tname, "ext", n), 1.0, (tname, "ext", "n100"))
        return Spec(cols, truth, names)
    i64_lo, i64_hi = TYPES["int"][1:]
    pool = [i64_lo, i64_hi, 0, -1] + _draw(rng, -(1 << 40), 1 << 40, 20)
    add(OBJ_INT, ENC_CS_INT_DICT, [pool[int(i)] for i in rng.integers(0, len(pool), size=n)], 0.10, ("int_dict", "pool", "n10"))
    upool = [(1 << 64) - 1, 1 << 63, 0] + _draw(rng, 0, 1 << 20, 9)
    add(OBJ_UINT64, ENC_CS_INT_DICT, [upool[int(i)] for i in rng.integers(0, len(upool), size=n)], 0.0, ("int_dict", "upool", "n0"))
    dom = [-777 if i % 23 else int(rng.integers(-5, 5)) for i in range(n)]        # const ref: <= 10 % exceptions (NULL among them)
    add(OBJ_INT, ENC_CS_INT_DICT, dom, 0.02, ("int_dict", "const_ref", "n2"))
    add(OBJ_INT, ENC_CS_INT_DICT, [5] * n, 1.0, ("int_dict", "null", "n100"))
    add(OBJ_VARCHAR, ENC_CS_STRING, strings(rng, n, 0, 3), 0.10, ("string", "tiny", "n10"))      # empty strings + NULL: bitmap
    add(OBJ_VARCHAR, ENC_CS_STRING, strings(rng, n, 1, 40), 0.0, ("string", "mid", "n0"))
    add(OBJ_VARCHAR, ENC_CS_STRING, strings(rng, n, 400, 1000), 0.10, ("string", "big", "n10"))  # > 65535 bytes per block
    add(OBJ_VARCHAR, ENC_CS_STRING, strings(rng, n, 1, 9), 1.0, ("string", "null", "n100"))
    words = strings(rng, 40, 0, 30)
    add(OBJ_VARCHAR, ENC_CS_STR_DICT, strings(rng, n, 0, 0, words), 0.10, ("str_dict", "var", "n10"))
    add(OBJ_VARCHAR, ENC_CS_STR_DICT, strings(rng, n, 0, 0, [w.ljust(16, b"_")[:16] for w in words[:12]]), 0.0, ("str_dict", "fix", "n0"))
    add(OBJ_VARCHAR, ENC_CS_STR_DICT, [b"dominant" if i % 23 else words[i % 40] for i in range(n)], 0.0, ("str_dict", "const_ref", "n0"))
    add(OBJ_VARCHAR, ENC_CS_STR_DICT, strings(rng, n, 1, 9), 1.0, ("str_dict", "null", "n100"))
    return Spec(cols, truth, names)


@functools.lru_cache(maxsize=None)
def column_table(mode, rpb, group):
    return encode_with(mode, column_spec(group, ROWS[rpb]).cols, rpb)


def block_rows(table):
    return [int(table.block(i)[16:20].view(np.uint32)[0]) for i in range(table.n_blocks)]


def int_form(obj, cells):
    """(NULL bitmap, base, NULL replacement, stored width) the writer gives a block of a CS_INTEGER column (ObIntegerColumnEncoder
    stream meta: sstable_writer.cpp build_cs); base and replacement as 64-bit images"""
    bits = 8 * STORE_SIZE[obj]
    mask = (1 << bits) - 1
    live = [c for c in cells if c is not None]
    has_null, bitmap, rep = len(live) < len(cells), False, None
    if obj in SIGNED:
        tmin, tmax = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        nmin, nmax = (min(live), max(live)) if live else (0, 0)
        if has_null:
            if nmin == 0 and nmax == tmax:
                nmin = rep = -1
            elif nmin in (0, tmin) and nmax != tmax:
                nmax = rep = nmax + 1
            elif nmin == tmin:
                bitmap = True
            else:
                nmin = rep = nmin - 1
        base = nmin if nmin < 0 else None
        top = nmax - nmin if base is not None else nmax
    else:
        live = [c & mask for c in live]
        nmin, nmax = (min(live), max(live)) if live else (0, 0)
        if has_null:
            if nmin == 0 and nmax == mask:
                bitmap = True
            elif nmin == 0:
                nmax = rep = nmax + 1
            else:
                nmin = rep = nmin - 1
        base, top = None, nmax
    width = 1 if top <= 0xFF else 2 if top <= 0xFFFF else 4 if top <= 0xFFFFFFFF else 8
    m64 = (1 << 64) - 1
    return bitmap, None if base is None else base & m64, None if rep is None else rep & m64, width


def int_form_of_block(block, c):
    """int_form as the block's CS column header and stream meta state it"""
    hs = int(block[4:8].view(np.uint32)[0])
    _, _, wtag, at, _, _ = next(s for s in stream_layout(block) if s[0] == c)
    _, base, rep = stream_meta(block, at)
    return bool(block[hs + 12 + 4 * c + 2] & 0x02), base, rep, 1 << wtag


def form_label(obj, cells):
    """which of the writer's ways int_form takes for a block"""
    bitmap, base, rep, _ = int_form(obj, cells)
    if bitmap:
        return "bitmap"
    if rep is None:
        return "plain" if base is None else "base"
    if rep == (1 << 64) - 1 and base == rep:
        return "minus1"                        # 0 and the type maximum present: NULL is -1, the base
    live = [c for c in cells if c is not None]
    return "above" if not live or rep == (max(live) + 1) & ((1 << 64) - 1) else "below"


def block_starts(table):
    return np.concatenate([[0], np.cumsum(block_rows(table))]).astype(np.int64)


def oracle_cells(blk, spec, c):
    """every cell of column c of an oracle block, as the column's own values"""
    rid = np.arange(blk.row_count, dtype=np.int32)
    if spec.is_str(c):
        return [blk.cell(c, r) for r in range(blk.row_count)]
    dl = datum_len(spec.obj[c])
    d, nulls, _ = blk.get_rows_fixed(c, rid, elem_len=dl)
    vals = d.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[dl])[:blk.row_count].tolist()
    isnull = (nulls[rid // 64] >> (rid % 64).astype(np.uint64)) & np.uint64(1)
    return [None if z else oracle_value(spec.obj[c], v) for v, z in zip(vals, isnull.tolist())]


def column_filters(spec):
    """(column, filter, rows the model selects) per column: BT over the middle half of its values and NU for integer columns,
    EQ on a value it holds for string columns"""
    import oceanbase_b200 as ob
    out = []
    for c, col in enumerate(spec.truth):
        if spec.is_str(c):
            k = next((x for x in col if x is not None), b"absent")
            out.append((c, ob.White(c, EQ, (k,)), [i for i, x in enumerate(col) if x == k]))
            continue
        live = sorted(x for x in col if x is not None)
        lo, hi = (live[len(live) // 4], live[3 * len(live) // 4]) if live else (0, 0)
        out.append((c, ob.White(c, BT, (lo, hi)), [i for i, x in enumerate(col) if x is not None and lo <= x <= hi]))
        out.append((c, ob.White(c, NU, ()), [i for i, x in enumerate(col) if x is None]))
    return out


def selected_rows(starts, sel_offset, row_ids):
    """the batch-wide row numbers of a scan's selected rows"""
    block = np.searchsorted(sel_offset, np.arange(len(row_ids)), side="right") - 1
    return (starts[block] + row_ids).tolist()


@pytest.mark.parametrize("mode,rpb", COLUMN_TABLES)
@pytest.mark.parametrize("group", GROUPS)
def test_column_matrix_headers_cells_and_filters(mode, rpb, group):
    spec = column_spec(group, ROWS[rpb])
    table, raw = column_table(mode, rpb, group), column_table(1, rpb, group)
    rows, starts = block_rows(table), block_starts(table)
    assert int(starts[-1]) == spec.n and table.n_blocks == raw.n_blocks
    forms, coded = set(), 0
    for i, nr in enumerate(rows):
        blk = table.block(i)
        hs = int(blk[4:8].view(np.uint32)[0])
        coded += len(coded_streams(blk))
        t = ora.cs_transform(blk)
        assert np.array_equal(t[hs:], raw.block(i)[hs:]), (MODES[mode], rpb, group, i)
        b = ora.Block(t)
        for c in range(len(spec.cols)):
            cells = spec.truth[c][starts[i]:starts[i] + nr]
            assert blk[hs + 12 + 4 * c + 1] == HEADER_TYPE[spec.enc[c]], spec.names[c]
            if spec.enc[c] == ENC_CS_INTEGER:
                assert int_form_of_block(blk, c) == int_form(spec.obj[c], cells), (spec.names[c], i)
                forms.add(form_label(spec.obj[c], cells))
            assert oracle_cells(b, spec, c) == cells, (MODES[mode], rpb, group, spec.names[c], i)
    if group != "dict_str" and rpb > 1:      # unsigned columns take no base
        assert forms == {"plain", "bitmap", "above", "below"} | ({"base", "minus1"} if group == "signed" else set()), forms
    if group == "dict_str" and rpb > 1:
        name = {n: c for c, n in enumerate(spec.names)}
        attrs = lambda c: int(table.block(0)[64 + 12 + 4 * c + 2])       # noqa: E731
        assert attrs(name[("string", "tiny", "n10")]) & 0x02              # empty strings and NULLs: a NULL bitmap
        assert not attrs(name[("string", "big", "n10")]) & 0x03           # variable length, NULL as zero length
        assert attrs(name[("str_dict", "fix", "n0")]) & 0x01              # fixed length: no offsets stream
        ends = {name[("string", n, r)] for n, r in (("tiny", "n10"), ("mid", "n0"), ("big", "n10"))}
        widths = {1 << s[2] for s in stream_layout(table.block(0)) if s[0] in ends and s[1] is not None}
        assert widths == {1, 2, 4} or rpb != 129, widths                  # END offsets of one, two and four bytes
    assert coded > 0, MODES[mode]
    # the oracle's filters over the restated blocks select the model's rows
    restated = ora.cs_transform_table(table)
    for c, f, want in column_filters(spec):
        res = ora.scan_table(restated, f, [c], [spec.is_str(c)], [8])
        assert selected_rows(starts, res["sel_offset"], res["row_ids"]) == want, (MODES[mode], rpb, group, spec.names[c], f)


# ---- 3. END offsets the restatement widens -------------------------------------------------------------------------------------
def offsets_width_tag(block):
    hs = int(block[4:8].view(np.uint32)[0])
    offsets_len = int(block[hs + 6:hs + 10].view(np.uint32)[0])
    return int(block[len(block) - offsets_len + 3])


@functools.lru_cache(maxsize=None)
def widening_table(which):
    """(single-block table coded with DOUBLE_DELTA_ZIGZAG_RLE, RAW twin, spec): 'four' -- 9000 rows of an 8-byte column of
    constant steps and a column of runs, a coded block of a few KiB whose restatement needs four-byte END offsets; 'two' -- 40
    rows of the 8-byte column, one-byte END offsets coded, two-byte ones restated"""
    import oceanbase_b200 as ob
    n = 9000 if which == "four" else 40
    mono = [(1 << 40) + 1_000_003 * i for i in range(n)]
    cols = [ob.Column(OBJ_UINT64, ENC_CS_INTEGER, as_store(mono))]
    truth = [mono]
    if which == "four":
        small = [int(x) for x in np.repeat(np.random.default_rng(9).integers(-3, 4, size=n // 50), 50)]
        cols.append(ob.Column(OBJ_INT, ENC_CS_INTEGER, as_store(small)))
        truth.append(small)
    return encode_with(2, cols, n), encode_with(1, cols, n), Spec(cols, truth, [("mono",), ("small",)][:len(cols)])


@pytest.mark.parametrize("which,tags", [("four", (1, 2)), ("two", (0, 1))])
def test_restatement_widens_the_end_offsets(which, tags):
    table, raw, spec = widening_table(which)
    blk = table.block(0)
    t = ora.cs_transform(blk)
    assert (offsets_width_tag(blk), offsets_width_tag(t)) == tags
    if which == "four":
        assert blk.size < 4 << 10 and t.size > 0xFFFF, (blk.size, t.size)
    assert np.array_equal(t[64:], raw.block(0)[64:])
    b = ora.Block(t)
    for c in range(len(spec.cols)):
        assert oracle_cells(b, spec, c) == spec.truth[c]
