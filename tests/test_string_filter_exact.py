"""String white filters, string projection and string skip-index verdicts against a plain model over Python bytes.

The project compares strings in binary collation only (DESIGN 3.8 and 8): memcmp over the common length, then the shorter string
first -- Python's own bytes order. NULL never passes a comparison, NE included; only NU / NN see NULL. A NULL constant makes EQ, NE,
LT, LE, GT, GE and BT select nothing; NULL constants inside IN are skipped, and an IN of only NULLs selects nothing. BT is inclusive
and selects nothing when lo > hi.

CPU half: the tables tests/test_gpu_string_filter_exact.py scans are what they claim to be -- every string codec the writer takes,
VARCHAR and CHAR, 0 %, 10 % and 100 % NULL -- the oracle decodes every cell back to the generated value, the column header shows the
intended codec, store and sorted flag, the oracle's white filters and trees select exactly the model's rows, and the oracle's
skip-index verdicts are sound under the model. The value pools and constants each target one edge of the device's string paths:
bytes >= 0x80 and NUL (signed-char compares, the __ffsll byte pick of str_cmp), strings equal in their first 8 bytes (the
(length, first 8 bytes) equality screen and the tail compare), lengths and first bytes that alias mod 64 (the two 64-bit screens of
an EQ / NE / IN leaf), IN lists whose constants clash under every hash multiplier, and the 48-constant / 768-byte constant limits."""
import functools

import numpy as np
import pytest

import oracle_binding as ora

EQ, LE, LT, GE, GT, NE, BT, IN, NU, NN = range(10)      # OBGPU_WHITE_OP_*
CMP_OPS = (EQ, NE, LT, LE, GT, GE)
U, T, F = 0, 1, 2                                        # skip-index verdicts: uncertain, always true, always false
OBJ_INT, OBJ_VARCHAR, OBJ_CHAR = 5, 22, 23
ENC_RAW, ENC_DICT, ENC_RLE, ENC_CONST = 0, 1, 2, 3
ENC_STRING_DIFF, ENC_HEX, ENC_STRING_PREFIX, ENC_COLUMN_EQUAL, ENC_COLUMN_SUBSTR = 5, 6, 7, 8, 9
ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STRING, ENC_CS_STR_DICT = 16, 17, 18, 19
MAX_PARAMS, PARAM_HEAP = 48, 768                         # kMaxParams, kParamHeap: a filter beyond them is OBGPU_NOT_SUPPORTED
N_ROWS, RPB = 1197, 133                                  # 9 full blocks
# row number (RAW), 0..99 (DICT: an integer leaf a stage record serves), the string column under test, a second string column
K, M, S, TCOL = range(4)


# ---- the model ------------------------------------------------------------------------------------------------------------
def leaf(op, cells, params):
    """verdict per cell (bytes or None; ints work the same way) of one white filter"""
    if op == NU:
        return [c is None for c in cells]
    if op == NN:
        return [c is not None for c in cells]
    if op == IN:
        ks = {p for p in params if p is not None}
        return [c is not None and c in ks for c in cells]
    if any(p is None for p in params):
        return [False] * len(cells)
    if op == BT:
        lo, hi = params
        return [c is not None and lo <= c <= hi for c in cells]
    k = params[0]
    f = {EQ: lambda c: c == k, NE: lambda c: c != k, LT: lambda c: c < k, LE: lambda c: c <= k, GT: lambda c: c > k,
         GE: lambda c: c >= k}[op]
    return [c is not None and f(c) for c in cells]


def model(expr, cols):
    """rows (verdict per row) of a filter tree; cols[c]: the cells of store column c"""
    if hasattr(expr, "children"):
        parts = [model(e, cols) for e in expr.children]
        fold = all if type(expr).__name__ == "And" else any
        return [fold(v) for v in zip(*parts)]
    return leaf(expr.op, cols[expr.col], tuple(expr.params))


def skip_sound(verdict, passed):
    """a skip-index verdict over a block whose cells the model passes as `passed`: FALSE -- no cell passes; TRUE -- every cell
    passes (for a comparison that also means the block holds no NULL)"""
    return verdict == U or (verdict == F and not any(passed)) or (verdict == T and all(passed))


# ---- the equality screens of an EQ / NE / IN leaf, restated from build_params (obgpu_scan.cu) -----------------------------
def str_eq_slot(pre, n, m):
    mult = (0xD6E8FEB86659FD93 + 2 * m * 0x9E3779B97F4A7C15) % (1 << 64)
    return ((((pre ^ ((n * 0x9E3779B97F4A7C15) % (1 << 64))) * mult) % (1 << 64)) >> 58)


def prefix8(s):
    return int.from_bytes(s[:8].ljust(8, b"\0"), "little")


def hash_multiplier(consts):
    """the multiplier index build_params gives a leaf's non-NULL constants (its hash-slot screen), None: the first-byte screen"""
    ks = [k for k in consts if k is not None]
    if not 1 <= len(ks) <= 32:
        return None
    for m in range(8):
        slots = [str_eq_slot(prefix8(k), len(k), m) for k in ks]
        if len(set(slots)) == len(slots):
            return m
    return None


def heap_bytes(consts):
    return sum((len(k) + 7) // 8 * 8 for k in consts if k is not None)


# ---- value pools ----------------------------------------------------------------------------------------------------------
def byte_pool(lengths=(16, 24)):
    """0x00 / 0x7F / 0x80 / 0xFF at positions 0, 7, 8, 15 and last: signed-char compares and the byte str_cmp picks"""
    out = []
    for n in lengths:
        for pos in sorted({0, 7, 8, 15, n - 1}):
            for b in (0x00, 0x7F, 0x80, 0xFF):
                s = bytearray(b"q" * n)
                s[pos] = b
                out.append(bytes(s))
    return out


LONG = bytes((0x30 + 7 * i) & 0xFF for i in range(300))             # bytes >= 0x80 from offset 12 on
LENGTHS = (0, 1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 300)   # one- and two-byte var offsets; > 255 bytes
LEN_POOL = [LONG[:n] for n in LENGTHS]
SHARED = [b"prefix08\x01tail", b"prefix08\x02tail", b"prefix08\x01tai\x80",       # same first 8 bytes and length, tails differ
          b"abcdefgh", b"abcdefgh\x00", b"abc", b"abc\x00"]                        # differ only in length
ALIAS67 = b"ali" + b"\0" * 5 + b"Z" * 59
ALIASES = [b"ali", ALIAS67, b"\x01fb", b"\x41fb", b"\x81fb", b"\xc1fb"]           # length 3 / 67 and first bytes alias mod 64
EDGE = list(dict.fromkeys(byte_pool() + LEN_POOL + SHARED + ALIASES))
FIX16 = list(dict.fromkeys(byte_pool((16,)) + [(b"prefix08" + t).ljust(16, b"_") for t in (b"\x01tail", b"\x02tail", b"\x01tai\x80")] +
                           [bytes([b]) + b"f" * 15 for b in (0x01, 0x41, 0x81, 0xC1)]))
HEX_ALPHA = bytes([0x00, 0x80, 0xFF, 0x7F, 0x01, 0x41, 0x81, 0xC1]) + b"abcdefgh"   # 16 bytes
GENERIC_CONSTS = [b"", b"\x00", b"\x80", b"\xff\xff\xff", b"abc", b"abc\x00", b"abcdefgh", b"abcdefgh\x00", b"prefix08\x01tail",
                  b"prefix08\x02tail", b"ali", ALIAS67, b"ali\x00\x00\x00\x00\x00", b"\x01fb", b"\x41fb", b"\x81fb", b"\xc1fb",
                  b"qqqqqqqq", b"q" * 16, LONG[:63], LONG[:64], LONG[:65], LONG[:127], LONG[:300], LONG[:299] + b"\x00"]


def clash_all_multipliers():
    """IN constants with distinct (length, first 8 bytes) that still clash under every one of the 8 multipliers: for each
    multiplier a colliding pair found by search -- the leaf keeps the first-byte screen"""
    out = []
    cand = [bytes([0x80 + i % 64]) + b"%06d" % i + bytes([0xFF - i % 7]) * (i % 5) for i in range(4000)]
    for m in range(8):
        seen = {}
        for c in cand:
            h = str_eq_slot(prefix8(c), len(c), m)
            if h in seen and c not in out and seen[h] not in out:
                out += [seen[h], c]
                break
            seen.setdefault(h, c)
    return out


CLASH = clash_all_multipliers()


def slot_distinct(pool, n, m=0):
    """n constants of pool, taken in order, whose slots under multiplier m are distinct: a 32-constant list that gets the hash
    slots (32 random constants in 64 slots almost always clash)"""
    out, used = [], set()
    for k in pool:
        h = str_eq_slot(prefix8(k), len(k), m)
        if h not in used:
            out.append(k)
            used.add(h)
        if len(out) == n:
            return out
    raise AssertionError("pool too small")


# ---- tables ---------------------------------------------------------------------------------------------------------------
# codec -> (encoding, value shape, header type, fixed store, sorted dictionary); None: not read from the header
CODECS = {
    "raw_var": (ENC_RAW, "edge", 0, False, None),
    "raw_fix": (ENC_RAW, "fix16", 0, True, None),
    "dict_var": (ENC_DICT, "edge", 1, False, False),
    "dict_fix": (ENC_DICT, "fix16", 1, True, True),
    "rle": (ENC_RLE, "runs", 2, None, None),
    "const": (ENC_CONST, "const", 3, None, None),
    "const_exc": (ENC_CONST, "const_exc", 3, None, None),
    "hex": (ENC_HEX, "hex", 6, None, None),
    "string_diff": (ENC_STRING_DIFF, "diff", 5, None, None),
    "string_prefix": (ENC_STRING_PREFIX, "prefix", 7, None, None),
    "column_equal": (ENC_COLUMN_EQUAL, "equal", 8, None, None),
    "column_substr": (ENC_COLUMN_SUBSTR, "substr", 9, None, None),
    "cs_string_var": (ENC_CS_STRING, "edge", 1, False, None),
    "cs_string_fix": (ENC_CS_STRING, "fix16", 1, True, None),
    "cs_str_dict_var": (ENC_CS_STR_DICT, "edge", 3, False, None),
    "cs_str_dict_fix": (ENC_CS_STR_DICT, "fix16", 3, True, None),
    "cs_str_dict_var_constref": (ENC_CS_STR_DICT, "const_exc", 3, False, None),
    "cs_str_dict_fix_constref": (ENC_CS_STR_DICT, "const_exc16", 3, True, None),
}
NULL_RATES = {"n0": 0.0, "n10": 0.10, "n100": 1.0}
OBJ_TYPES = {"varchar": OBJ_VARCHAR, "char": OBJ_CHAR}


def is_cs(codec):
    return CODECS[codec][0] >= 16


def all_null_encoding(codec):
    """The writer refuses an all-NULL column for codecs that need at least one value (DICT, RLE, HEX_PACKING, STRING_DIFF,
    STRING_PREFIX: no dictionary entry, no alphabet, no common bytes, no prefix) and for a span column whose every cell is an
    exception; such a column is CONST of NULL (PAX) there. CS string columns take an all-NULL column as they are."""
    enc = CODECS[codec][0]
    if enc in (ENC_DICT, ENC_RLE, ENC_HEX, ENC_STRING_DIFF, ENC_STRING_PREFIX):
        return ENC_CONST
    return enc


def gen_strings(rng, shape, n):
    if shape in ("edge", "fix16"):
        pool = EDGE if shape == "edge" else FIX16
        return [pool[i] for i in rng.integers(0, len(pool), size=n).tolist()]
    if shape == "runs":
        out = []
        while len(out) < n:
            out += [EDGE[int(rng.integers(0, len(EDGE)))]] * int(rng.integers(1, 9))
        return out[:n]
    if shape in ("const", "const_exc", "const_exc16"):
        # one value, and for the _exc shapes one exception every 37 rows (fewer than 10 % of every block), of other lengths than
        # the value's (a var store) or of the same length (_exc16: a fixed store)
        value, pool = (FIX16[3], FIX16[4:]) if shape == "const_exc16" else (b"abcdefgh", [v for v in EDGE[36:] if len(v) != 8])
        out = [value] * n
        if shape != "const":
            for i in range(11, n, 37):
                out[i] = pool[(i // 37) % len(pool)]
        return out
    if shape == "hex":
        lens = (0, 1, 7, 8, 9, 15, 16, 17, 40, 63, 64, 65)
        a = np.frombuffer(HEX_ALPHA, dtype=np.uint8)
        return [bytes(a[rng.integers(0, 16, size=lens[int(rng.integers(0, len(lens)))])]) for _ in range(n)]
    if shape == "diff":             # 24 bytes; high bytes in the common part (0..2, 12) and in the differing positions (3, 8, 9, 15)
        tmpl = bytearray(b"\xff\x80\x00" + b"d" * 9 + b"\xc1" + b"e" * 11)
        out = []
        for _ in range(n):
            s = bytearray(tmpl)
            for pos in (3, 8, 9, 15):
                s[pos] = (0x00, 0x7F, 0x80, 0xFF, 0x61)[int(rng.integers(0, 5))]
            out.append(bytes(s))
        return out
    if shape == "prefix":           # high bytes in the shared prefixes and in the rests
        pres = [b"\x81pre\xff/", b"\x01pre\x00/", b"Apre\x80/x", b"\xc1", b"\x00\x00\x00\x00\x00\x00\x00\x00zz"]
        rest = bytes([0x00, 0x7F, 0x80, 0xFF]) + b"rst"
        return [pres[int(rng.integers(0, len(pres)))] + bytes(rng.choice(np.frombuffer(rest, dtype=np.uint8),
                                                                          size=int(rng.integers(0, 13)))) for _ in range(n)]
    raise ValueError(shape)


def null_mask(rng, shape, n, rate):
    if rate >= 1.0:
        return np.ones(n, dtype=np.uint8)
    m = np.zeros(n, dtype=np.uint8)
    if rate == 0.0:
        return m
    if shape.startswith("const"):   # NULL is an exception of a CONST column (and of a const ref) too: a fixed stride
        m[7::25] = 1
        return m
    if shape == "fix16":            # a fixed store stays fixed while the NULL cells' padding costs less than var offsets would
        m[3::11] = 1
        return m
    return (rng.random(n) < rate).astype(np.uint8)


def with_nulls(values, mask):
    return [None if z else v for v, z in zip(values, mask.tolist())]


class Spec:
    """one generated table: the writer's columns and the true cell (bytes, int or None) of every row of every column"""

    def __init__(self, cols, truth, s_encoding, obj):
        self.cols, self.truth, self.s_encoding, self.obj = cols, truth, s_encoding, obj
        self.n = len(truth[0])


@functools.lru_cache(maxsize=None)
def spec_of(codec, tname, nname, n=N_ROWS, seed=0):
    import oceanbase_b200 as ob
    enc, shape, _, _, _ = CODECS[codec]
    obj = OBJ_TYPES[tname]
    rate = NULL_RATES[nname]
    rng = np.random.default_rng(100 * list(CODECS).index(codec) + 10 * list(OBJ_TYPES).index(tname) + list(NULL_RATES).index(nname) + seed)
    ienc = ENC_CS_INTEGER if is_cs(codec) else ENC_RAW
    denc = ENC_CS_INT_DICT if is_cs(codec) else ENC_DICT
    senc = ENC_CS_STRING if is_cs(codec) else ENC_RAW
    k = list(range(n))
    m = [int(x) for x in rng.integers(0, 100, size=n).tolist()]
    tvals = gen_strings(rng, "edge", n)
    nt = (rng.random(n) < 0.10).astype(np.uint8)
    if shape in ("equal", "substr"):
        ns = null_mask(rng, "edge", n, rate)
        nt = ns.copy()                      # both cells NULL: not an exception of the span column
        if shape == "equal":            # the column equals the second column but at one row in 37
            svals = list(tvals)
            for i in range(5, n, 37):
                svals[i] = EDGE[(i + 1) % len(EDGE)] if EDGE[(i + 1) % len(EDGE)] != tvals[i] else EDGE[(i + 2) % len(EDGE)]
        else:                           # a substring of the second column's value in the same row
            tvals = [v + b"\x80sub\xff" + bytes([i % 251]) for i, v in enumerate(tvals)]
            svals = [v[1:1 + (i % 11)] for i, v in enumerate(tvals)]
    else:
        svals = gen_strings(rng, shape, n)
        ns = null_mask(rng, shape, n, rate)
    s_enc = all_null_encoding(codec) if rate >= 1.0 else enc
    cols = [ob.Column(OBJ_INT, ienc, np.array(k, dtype=np.int64)), ob.Column(OBJ_INT, denc, np.array(m, dtype=np.int64)),
            ob.Column(obj, s_enc, svals, nulls=ns, ref_col=TCOL),
            # a span column refers to a column of its own type
            ob.Column(obj if shape in ("equal", "substr") else OBJ_VARCHAR, senc, tvals, nulls=nt)]
    return Spec(cols, [k, m, with_nulls(svals, ns), with_nulls(tvals, nt)], s_enc, obj)


@functools.lru_cache(maxsize=None)
def table_of(codec, tname, nname, rpb=RPB):
    import oceanbase_b200 as ob
    return ob.encode_table(spec_of(codec, tname, nname).cols, rpb)


MATRIX = [(c, t, nn) for c in CODECS for t in OBJ_TYPES for nn in NULL_RATES]
MATRIX_IDS = ["-".join(x) for x in MATRIX]


# ---- constants and filters ------------------------------------------------------------------------------------------------
def consts_of(spec):
    """the generic edge constants + a few of the column's own values, each also with its last byte bumped (absent values)"""
    present = sorted({v for v in spec.truth[S] if v is not None})
    picks = [present[i] for i in np.linspace(0, len(present) - 1, num=min(6, len(present))).astype(int).tolist()] if present else []
    bumped = [p[:-1] + bytes([(p[-1] + 1) & 0xFF]) for p in picks if p]
    return list(dict.fromkeys(GENERIC_CONSTS + picks + bumped))


def in_lists(spec):
    """name -> IN constants; each list targets one screen or limit"""
    cs = consts_of(spec)
    present = [v for v in dict.fromkeys(spec.truth[S]) if v is not None]
    p0 = next((v for v in present if len(v) <= 64), b"abc")      # three copies of it stay inside the constant heap
    # constants of <= 16 bytes (48 of them fit the heap), absent ones last
    pool = [k for k in dict.fromkeys(present + cs + EDGE + [b"k%02d\x80" % i for i in range(64)]) if len(k) <= 16]
    return {
        "in1": [p0],
        "in2": [p0, b"nowhere\x80"],
        "in32": slot_distinct(pool, 32),
        "in33": slot_distinct(pool, 32) + [k for k in pool if k not in slot_distinct(pool, 32)][:1],   # > 32: first-byte screen
        "in_clash_pair": [b"prefix08\x01tail", b"prefix08\x02tail", p0],    # equal (length, first 8 bytes): clash everywhere
        "in_clash_search": CLASH + [p0],
        "in_dup_null_empty": [p0, p0, None, b"", b"absent\xff", None, p0],
        "in_only_null": [None, None],
        "in48": pool[:MAX_PARAMS],
        "in_heap_767": [LONG[:255], LONG[:256], b"\xff" * 8 + LONG[:248]],     # 767 bytes, 768 padded: the whole heap
    }


def leaves(spec):
    """(name, filter) of every single-leaf filter a table is checked with"""
    import oceanbase_b200 as ob
    cs = consts_of(spec)
    out = [("nu", ob.White(S, NU, ())), ("nn", ob.White(S, NN, ()))]
    for op in CMP_OPS:
        out += [("%d:%r" % (op, c[:12]), ob.White(S, op, (c,))) for c in cs]
        out.append(("%d:null" % op, ob.White(S, op, (None,))))
    for lo, hi in ((b"", b"\xff" * 4), (b"abc", b"abcdefgh"), (b"abcdefgh", b"abc"), (b"\x80", b"\xff"), (b"abc\x00", b"abc\x00"),
                   (LONG[:63], LONG[:65]), (b"\x00", b"\x7f\xff"), (None, b"\xff"), (b"q" * 8, b"q" * 16)):
        out.append(("bt:%r:%r" % (lo and lo[:8], hi and hi[:8]), ob.White(S, BT, (lo, hi))))
    out += [(name, ob.White(S, IN, tuple(ks))) for name, ks in in_lists(spec).items()]
    return out


def trees(spec):
    """(name, filter) of the trees: the survivor path (a selective integer leaf first, then string leaves), an OR of a string IN
    and integer leaves, two string leaves on one column"""
    import oceanbase_b200 as ob
    present = [v for v in dict.fromkeys(spec.truth[S]) if v is not None] or [b"abc"]
    a, b = sorted(present)[len(present) // 4], sorted(present)[3 * len(present) // 4]
    W = ob.White
    return [
        ("and_m_eq", ob.And([W(M, EQ, (7,)), W(S, EQ, (present[0],))])),
        ("and_m_in", ob.And([W(M, LT, (3,)), W(S, IN, (present[0], b"prefix08\x02tail", LONG[:65], b""))])),
        ("and_m_ne", ob.And([W(M, EQ, (11,)), W(S, NE, (present[-1],))])),
        ("and_m_nu", ob.And([W(M, LT, (3,)), W(S, NU, ())])),
        ("and_m_nn", ob.And([W(M, LT, (3,)), W(S, NN, ())])),
        ("and_m_lt", ob.And([W(M, EQ, (5,)), W(S, LT, (b,))])),
        ("or_in_int", ob.Or([W(S, IN, (present[0], present[-1], b"\x81fb")), W(K, LT, (40,)), W(M, EQ, (3,))])),
        ("and_two_str", ob.And([W(S, GE, (a,)), W(S, LT, (b,))])),
        ("and_two_str_eq", ob.And([W(S, NE, (a,)), W(S, IN, (a, b, present[0]))])),
        ("or_eq_nu", ob.Or([W(S, EQ, (b,)), W(S, NU, ())])),
        ("and_str_t", ob.And([W(S, GT, (b"\x7f",)), W(TCOL, LE, (b"prefix08\x01tail",))])),
        ("and_48_params", ob.And([W(S, IN, SHORT49[:MAX_PARAMS - 1]), W(S, NE, (present[0],))])),     # kMaxParams over the tree
    ]


SHORT49 = tuple(b"k%02d\x80" % i for i in range(MAX_PARAMS + 1))     # 49 constants of 4 bytes: 392 padded heap bytes


def over_limits(spec):
    """(name, filter, limit) the device refuses with OBGPU_NOT_SUPPORTED when it builds the scan parameters: "params" -- more than
    kMaxParams constants over the whole tree, with the heap well inside kParamHeap; "heap" -- more than kParamHeap bytes of padded
    string constants, with few constants. The oracle has no such limits."""
    import oceanbase_b200 as ob
    W = ob.White
    return [("in49", W(S, IN, SHORT49), "params"),
            ("and_48_plus_1", ob.And([W(S, IN, SHORT49[:MAX_PARAMS]), W(S, NE, (b"abc",))]), "params"),
            ("in_heap_776", W(S, IN, (LONG[:256], LONG[:255] + b"\x00", LONG[:257])), "heap"),
            ("and_heap_776", ob.And([W(S, GE, (LONG[:256],)), W(S, LE, (LONG[:264],)), W(S, NE, (LONG[:249],))]), "heap")]


def tree_params(f):
    """the non-NULL constants of every leaf of a filter tree, as build_params counts them"""
    return [p for x in getattr(f, "children", [f]) for p in x.params if p is not None]


def selected(spec, expr):
    return [i for i, v in enumerate(model(expr, spec.truth)) if v]


# ---- what the writer wrote ------------------------------------------------------------------------------------------------
def header_facts(table, col):
    """per block (header type, fixed store or None, dictionary sorted flag or None) of one column"""
    img, off = np.asarray(table.image), np.asarray(table.offsets)
    out = []
    for b in range(table.n_blocks):
        o = int(off[b])
        hs = int(img[o + 4:o + 8].view(np.uint32)[0])
        n_cols = int(img[o + 10:o + 12].view(np.uint16)[0])
        if int(img[o + 20]) == 3:                   # CS_ENCODING_ROW_STORE: ObCSColumnHeader {version, type, attrs, obj_type}
            h = img[o + hs + 12 + 4 * col:o + hs + 16 + 4 * col]
            out.append((int(h[1]), bool(h[2] & 0x1), None))
            continue
        h = img[o + hs + 16 * col:o + hs + 16 * col + 16]
        fixed = bool(h[2] & 0x1) if h[1] == ENC_RAW else None
        srt = None
        if h[1] == ENC_DICT:                        # ObDictMetaHeader::attr_: FIX_LENGTH 0x1, IS_SORTED 0x2
            attr = int(img[o + hs + 16 * n_cols + int(h[8:12].view(np.uint32)[0]) + 8])
            fixed, srt = bool(attr & 0x1), bool(attr & 0x2)
        out.append((int(h[1]), fixed, srt))
    return out


def assert_headers(codec, nname, spec, table, store=True):
    """the writer chose the intended codec, store and sorted flag for the string column in every block, and a dictionary for the
    0..99 column (store=False: the codec only)"""
    enc, shape, htype, fixed, srt = CODECS[codec]
    assert {f[0] for f in header_facts(table, M)} == {2 if is_cs(codec) else ENC_DICT}
    facts = header_facts(table, S)
    if spec.s_encoding != enc:
        assert {f[0] for f in facts} == {ENC_CONST}
        return
    assert {f[0] for f in facts} == {htype}, facts
    if store and fixed is not None and NULL_RATES[nname] < 1.0:
        assert {f[1] for f in facts} == {fixed}, facts
    if store and srt is not None:
        assert {f[2] for f in facts} == {srt}, facts


def test_model_semantics():
    cells = [b"abc", None, b"abc\x00", b"ab\xff", b"", b"\x80"]
    assert leaf(LT, cells, (b"abc\x00",)) == [True, False, False, False, True, False]    # a prefix sorts first; 0xFF > 'c'
    assert leaf(NE, cells, (b"abc",)) == [False, False, True, True, True, True]          # NULL never passes NE
    assert leaf(NE, cells, (None,)) == [False] * 6 and leaf(BT, cells, (b"", None)) == [False] * 6
    assert leaf(IN, cells, (None, b"", None)) == [False, False, False, False, True, False]
    assert leaf(IN, cells, (None,)) == [False] * 6
    assert leaf(BT, cells, (b"b", b"a")) == [False] * 6 and leaf(BT, cells, (b"", b"")) == [False, False, False, False, True, False]
    assert leaf(NU, cells, ()) == [False, True, False, False, False, False]
    assert skip_sound(F, [False, False]) and not skip_sound(F, [True, False]) and not skip_sound(T, [True, False])


def test_screens_each_list_targets():
    """which equality screen build_params gives each IN list (the hash slots need 1..32 constants distinct under a multiplier)"""
    spec = spec_of("dict_var", "varchar", "n10")
    lists = in_lists(spec)
    for name in ("in1", "in2", "in32", "in_heap_767"):
        assert hash_multiplier(lists[name]) is not None, name
    # duplicates clash with themselves: the duplicated list keeps the first-byte screen too
    for name in ("in33", "in48", "in_clash_pair", "in_clash_search", "in_dup_null_empty", "in_only_null"):
        assert hash_multiplier(lists[name]) is None, name
    assert len(CLASH) <= 32 and len({(len(k), prefix8(k)) for k in CLASH}) == len(CLASH)
    assert len(lists["in32"]) == 32 and len(lists["in33"]) == 33 and len(lists["in48"]) == MAX_PARAMS
    assert 760 < heap_bytes(lists["in_heap_767"]) <= PARAM_HEAP and sum(map(len, lists["in_heap_767"])) == 767
    assert all(heap_bytes(ks) <= PARAM_HEAP and len(ks) <= MAX_PARAMS for ks in lists.values())     # the device takes each list
    # each refused filter breaks exactly the limit it is named for, and the accepted 48-constant tree breaks neither
    for name, f, limit in over_limits(spec):
        ks = tree_params(f)
        assert (len(ks) > MAX_PARAMS, heap_bytes(ks) > PARAM_HEAP) == (limit == "params", limit == "heap"), name
    ks = tree_params(dict(trees(spec))["and_48_params"])
    assert len(ks) == MAX_PARAMS and heap_bytes(ks) <= PARAM_HEAP
    # the screens' aliases are really in the pools: lengths 3 / 67 and 1 / 65, first bytes 0x01 / 0x41 / 0x81 / 0xC1
    assert {3, 67, 1, 65} <= {len(v) for v in EDGE} and {v[0] & 63 for v in (b"\x01", b"\x41", b"\x81", b"\xc1")} == {1}


@pytest.mark.parametrize("codec,tname,nname", MATRIX, ids=MATRIX_IDS)
def test_table_inputs_and_oracle_filters(codec, tname, nname):
    spec = spec_of(codec, tname, nname)
    table = table_of(codec, tname, nname)
    # the oracle decodes every cell back to the generated value / NULL
    for b in range(table.n_blocks):
        blk = ora.Block(table.block(b))
        r0 = b * RPB
        for c in range(4):
            got = [blk.cell(c, r) for r in range(blk.row_count)]
            assert got == spec.truth[c][r0:r0 + blk.row_count], (b, c)
        ora.arena_reset()
    assert_headers(codec, nname, spec, table)
    if codec.endswith("constref") and NULL_RATES[nname] < 1.0:
        # the writer's const-ref rule (one ref covers all but <= 64 rows and fewer than 10 % of a block) holds in every block
        for b in range(table.n_blocks):
            cells = spec.truth[S][b * RPB:(b + 1) * RPB]
            top = max(cells.count(v) for v in set(cells))
            assert len(cells) == top or (len(cells) - top <= 64 and len(cells) - top < len(cells) * 10 // 100)
    # every IN list fits the device's constant limits (over_limits holds the ones that do not)
    assert all(heap_bytes(ks) <= PARAM_HEAP and len(ks) <= MAX_PARAMS for ks in in_lists(spec).values())
    # the oracle's filters and trees select exactly the model's rows
    for name, f in leaves(spec) + trees(spec) + [x[:2] for x in over_limits(spec)]:
        got = ora.scan_table(table, f, [K], [False], [8])
        assert got["data"][0].tolist() == selected(spec, f), name
    ora.arena_reset()


# ---- skip index ------------------------------------------------------------------------------------------------------------
SKIP_OPS = CMP_OPS + (BT, IN, NU, NN)


def skip_filters(spec):
    cs = consts_of(spec)
    import oceanbase_b200 as ob
    out = [ob.White(S, op, (c,)) for op in CMP_OPS for c in cs]
    out += [ob.White(S, BT, (lo, hi)) for lo, hi in ((b"", b"\x80"), (b"abc", b"abcdefgh"), (LONG[:40], LONG[:45]), (b"\x80", b"\xff"))]
    out += [ob.White(S, IN, tuple(ks)) for ks in in_lists(spec).values()] + [ob.White(S, NU, ()), ob.White(S, NN, ())]
    return out


def long_minmax_spec():
    """a table whose blocks' minimum and maximum are longer than 40 bytes, with high bytes inside the first 40: the writer stores
    40-byte prefixes"""
    import oceanbase_b200 as ob
    n = 4 * RPB
    rng = np.random.default_rng(5)
    heads = [b"\x80" * 3 + b"lo", b"\xff\x00" + b"hi", b"m\x7f"]
    vals = [heads[int(rng.integers(0, 3))] + bytes(rng.integers(0, 256, size=int(rng.integers(38, 60)), dtype=np.uint8))
            for _ in range(n)]
    ns = (rng.random(n) < 0.1).astype(np.uint8)
    cols = [ob.Column(OBJ_INT, ENC_RAW, np.arange(n, dtype=np.int64)), ob.Column(OBJ_INT, ENC_RAW, np.zeros(n, dtype=np.int64)),
            ob.Column(OBJ_VARCHAR, ENC_RAW, vals, nulls=ns), ob.Column(OBJ_VARCHAR, ENC_RAW, vals)]
    return Spec(cols, [list(range(n)), [0] * n, with_nulls(vals, ns), vals], ENC_RAW, OBJ_VARCHAR)


def hand_rows():
    """(cells of a block, aggregate row) pairs whose stored minimum / maximum is a prefix (is_prefix) that is a prefix of a
    constant, equals a constant, or is longer than a constant; the block's true cells are consistent with the prefixes"""
    import oceanbase_b200 as ob
    out = []
    for lo_real, hi_real, lo_pre, hi_pre in (
            (b"abc" + b"\x01" * 45, b"abc" + b"\xff" * 45, b"abc", b"abc"),              # prefix of the constant b"abcd"
            (b"abcd" + b"\x00" * 40, b"abcd" + b"\x90" * 40, b"abcd", b"abcd"),          # equals the constant b"abcd"
            (b"abcde\x80" + b"z" * 40, b"abcdf" + b"\x00" * 40, b"abcde\x80", b"abcdf"),  # longer than the constant b"abcd"
            (b"ab" + b"\x00" * 50, b"abcd" + b"\x7f" * 50, b"ab", b"abcd")):
        # with one NULL cell, and NULL-free (only there can a verdict be TRUE)
        for cells in ([lo_real, hi_real, lo_real + b"\x01", None], [lo_real, hi_real, lo_real + b"\x01", hi_real]):
            nc = cells.count(None).to_bytes(8, "little")
            out.append((cells, ob.agg_row_write([(S, 0, (lo_pre, True)), (S, 1, (hi_pre, True)), (S, 2, nc)])))
    return out


HAND_CONSTS = [b"abcd", b"abc", b"abcde", b"abcd\x00", b"abcd\xff", b"ab", b"abce", b"", b"\x80"]


def hand_filters():
    import oceanbase_b200 as ob
    out = [ob.White(S, op, (c,)) for op in CMP_OPS for c in HAND_CONSTS]
    out += [ob.White(S, BT, (lo, hi)) for lo in HAND_CONSTS[:4] for hi in HAND_CONSTS[:5]]
    out += [ob.White(S, IN, (b"abcd", b"abc")), ob.White(S, IN, (b"abcd\x00", None)), ob.White(S, NU, ()), ob.White(S, NN, ())]
    return out


SKIP_TABLES = [("dict_var", "varchar", "n10"), ("raw_var", "varchar", "n0"), ("string_prefix", "char", "n10"),
               ("cs_str_dict_fix", "varchar", "n10"), ("raw_var", "varchar", "n100")]


def skip_cases():
    """(spec, table rows cut per block, agg rows, agg offsets) of the tables the skip index is checked over"""
    import oceanbase_b200 as ob
    out = []
    for key in SKIP_TABLES:
        spec = spec_of(*key)
        rows, offs = ob.table_agg_rows(spec.cols, [S], RPB)
        out.append((key, spec, rows, offs))
    spec = long_minmax_spec()
    rows, offs = ob.table_agg_rows(spec.cols, [S], RPB)
    out.append((("long_minmax",), spec, rows, offs))
    return out


COL_TYPES = [OBJ_INT, OBJ_INT, OBJ_VARCHAR, OBJ_VARCHAR]


def test_skip_index_verdicts_are_sound():
    seen_prefix = False
    decided = 0
    for key, spec, rows, offs in skip_cases():
        for b in range((spec.n + RPB - 1) // RPB):
            row = rows[int(offs[b]):int(offs[b + 1])]
            cells = spec.truth[S][b * RPB:(b + 1) * RPB]
            mn, pre = ora.agg_row_read(row, S, 0)
            seen_prefix |= pre and len(mn) == 40 and max(mn) >= 0x80
            for f in skip_filters(spec):
                v = ora.skip_index_filter(row, len(cells), COL_TYPES, f)
                assert skip_sound(v, leaf(f.op, cells, tuple(f.params))), (key, b, f)
                decided += v != U
    assert seen_prefix and decided > 100
    verdicts = set()
    for cells, row in hand_rows():
        for f in hand_filters():
            v = ora.skip_index_filter(row, len(cells), COL_TYPES, f)
            assert skip_sound(v, leaf(f.op, cells, tuple(f.params))), (cells[0][:8], f)
            verdicts.add(v)
    assert verdicts == {U, T, F}        # the prefix rule is exercised on both certain sides
