"""The tables and cases of test_gpu_scan_plan.py, and the facts each case stands on, checked without a device.

Each case of the GPU file sits on one side of a limit of the scan planner (plan_scan, obgpu_scan.cu): a block row count, a
column's region or projection span, a dictionary size, a layout's shared-memory bytes. This module builds every table the GPU
file scans, reads those facts from the block bytes (the column headers and plans as the index kernel derives them), and
asserts that each case really sits where it claims. The GPU file imports its cases from here, so the two cannot drift apart.

Shared-memory limits are the H100's (227 KiB opt-in per block, of which the library keeps 1 KiB for static shared memory);
the GPU file recomputes them from the device it runs on and skips a pair the device's limit does not split.
"""
import functools
from dataclasses import dataclass, field
from typing import Callable, Optional, Sequence, Tuple

import numpy as np

import oracle_binding as ora

# numbering of obgpu_ctx_scan_plan (include/obgpu_scan.h)
NONE, PLANS, RECORDS, CODED, CTA, BITMAP = 0, 1, 2, 3, 4, 5                  # OBGPU_SCAN_COUNT_*
P_NONE, P_CTA, P_SPARSE, P_PLANS, P_RECORDS = 0, 1, 2, 3, 4                    # OBGPU_SCAN_PROJ_*
F_COMPACT, F_NO_STAGE, F_SPARSE = 1, 2, 4                                      # OBGPU_SCAN_PROJ_FLAG_*

H100_SMEM_OPTIN = 232448        # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SMEM_HEADROOM = 1024            # obgpu_ctx_create keeps this much for the kernels' static shared memory
WARPS = 4                       # warps per CTA of the scan kernels (kWarps)
COUNT_SPAN_CAP, PROJ_SPAN_CAP = 12288, 16384


def r16(v):
    return (v + 15) & ~15


def r128(v):
    return (v + 127) & ~127


# ---- facts from the block bytes ----------------------------------------------------------------------------------------------
def _u(s, o, n):
    return int.from_bytes(bytes(s[o:o + n]), "little")


def column_ranges(s, size, col):
    """(region, projection bytes, dictionary entries) of column col of one PAX block, as col_region / proj_ranges_bytes
    (scan_device.cuh) compute them: region = hi - lo of the 16-byte aligned, over-read padded byte range, or None for a
    column with no single region (CS blocks). Covers the encodings the tables below use: RAW (bit-packed, fixed, var-stored)
    and DICT."""
    s = bytes(s)
    if s[20] == 3:                       # CS_ENCODING_ROW_STORE: CS string bytes live outside any column region
        return None, None, 0
    hs, nc, rows = _u(s, 4, 4), _u(s, 8, 4) >> 16, _u(s, 16, 4)
    ext_bit, row_data_off = (s[21] >> 3) & 7, _u(s, 24, 4)
    ch = hs + 16 * col
    typ, attr, obj = s[ch + 1], s[ch + 2], s[ch + 3]
    offset, length = _u(s, ch + 8, 4), _u(s, ch + 12, 4)
    meta = hs + 16 * nc + offset
    is_str = obj in (22, 23)
    has_ext, fixed, bp = attr & 2, attr & 1, attr & 4
    ext_bits = (ext_bit if has_ext else 0) * rows
    ext_bit_off = meta * 8
    aligned = lambda a, b: ((b + 31) & ~15) - (a & ~15)
    if typ == 0:                          # RAW
        if bp:
            val_bit = meta * 8 + ext_bits
            a = (min(ext_bit_off, val_bit) if ext_bits else val_bit) >> 3
            b = (val_bit + rows * length + 7) >> 3
        elif fixed and is_str:            # K_FIXSTR: val_bit is a byte offset here
            data = meta + (ext_bits + 7) // 8
            a = ext_bit_off >> 3 if ext_bits else data
            b = data + rows * length
        elif fixed:
            val_bit = (meta + (ext_bits + 7) // 8) * 8
            a = (min(ext_bit_off, val_bit) if ext_bits else val_bit) >> 3
            b = (val_bit + rows * length * 8 + 7) >> 3
        else:                             # var-stored cells: the row data up to the block's end
            a, b = row_data_off, int(size)
        span = aligned(a, b)
        return span, span, 0
    assert typ == 1, f"column {col}: encoding {typ} is not modelled here"
    ref_size, count, dds, dattr = s[meta + 1], _u(s, meta + 2, 4), _u(s, meta + 6, 2), s[meta + 8]
    payload, dict_end, val_bit = meta + 9, meta + length, (meta + length) * 8
    stride = ref_size if bp else ref_size * 8
    refs_end = (val_bit + rows * stride + 7) >> 3
    span = aligned(payload, max(refs_end, dict_end))
    if not is_str:
        return span, span, count
    ref_lo, ref_hi = (val_bit >> 3) & ~15, (refs_end + 31) & ~15
    if dattr & 1:                         # fixed-length string entries: a cell's address is arithmetic, the refs suffice
        return span, ref_hi - ref_lo, count
    idx_lo, idx_hi = payload & ~15, (payload + count * dds + 31) & ~15
    if idx_hi < ref_lo or ref_hi < idx_lo:
        return span, (idx_hi - idx_lo) + (ref_hi - ref_lo), count
    return span, max(idx_hi, ref_hi) - min(idx_lo, ref_lo), count


@dataclass
class Facts:
    total_rows: int
    max_rows: int
    block_bytes: int                      # r128(largest 16-byte padded block + 16): a staged block (layout_project_cta)
    span: list                            # per column, max over the blocks (None: no single region)
    pspan: list
    max_dict: list                        # per column, largest dictionary + 2 (predicate bitset bits)


def table_facts(table, n_cols):
    span, pspan, dct = [0] * n_cols, [0] * n_cols, [0] * n_cols
    rows, big = [], 0
    for i in range(table.n_blocks):
        s, size = table.block(i), int(table.sizes[i])
        rows.append(ora.Block(s).row_count)
        big = max(big, r16(size))
        for c in range(n_cols):
            sp, ps, cnt = column_ranges(s, size, c)
            span[c] = None if sp is None or span[c] is None else max(span[c], sp)
            pspan[c] = None if ps is None or pspan[c] is None else max(pspan[c], ps)
            dct[c] = max(dct[c], cnt + 2 if cnt else 0)
    return Facts(sum(rows), max(rows), r128(big + 16), span, pspan, dct)


# ---- layouts, as layout_count_pipe / layout_project_pipe / layout_count_cta size them (records: stage records) ---------------
def count_pipe_bytes(f, filter_cols, n_slots, rec=False):
    """per-warp bytes of obgpu_count_pipe_kernel with no batch codes"""
    words_cap, rows_cap = (max(f.max_rows, 32) + 31) // 32, max(f.max_rows, 32)
    bitset = r16(n_slots * max((f.max_dict[c] + 31) // 32 for c in filter_cols) * 4) if n_slots else 0
    w = 3 * (64 + len(filter_cols) * (32 if rec else 96)) + 2 * (64 + sum(r16(f.span[c]) for c in filter_cols))
    w += r16(max(words_cap, 32) * 4) + r16(rows_cap * 2) + bitset + 16
    return r128(w) + 128


def proj_pipe_bytes(f, proj, rec):
    """per-warp bytes of obgpu_project_pipe_kernel over columns without run-length encoding"""
    words_cap, rows_cap = (max(f.max_rows, 32) + 31) // 32, max(f.max_rows, 32)
    region = r16((2 * 24 + 1) * 4) + r16(words_cap * 4) + sum(r16(f.pspan[c]) for c in proj)
    return r128(3 * (64 + max(len(proj), 1) * (64 if rec else 96)) + 2 * region + r16(rows_cap * 2) + 16)


def count_cta_bytes(f, filter_cols, n_slots):
    """per-warp bytes of obgpu_count_kernel"""
    words_cap = (max(f.max_rows, 32) + 31) // 32
    stage = max([f.span[c] for c in filter_cols if f.span[c] is not None and f.span[c] <= 24576] + [0])
    bitset = r16(n_slots * max((f.max_dict[c] + 31) // 32 for c in filter_cols) * 4) if n_slots else 0
    return r128(r16(96 * len(filter_cols)) + r16(words_cap * 4) + bitset + stage)


def compact(f, proj):
    """layout_project_cta stages the projected columns' regions alone"""
    return bool(proj) and all(f.span[c] is not None for c in proj) and sum(f.span[c] for c in proj) * 4 <= f.block_bytes * 3


def two_ctas(per_warp, max_smem):
    return per_warp * WARPS * 2 <= max_smem


H100_MAX_SMEM = H100_SMEM_OPTIN - SMEM_HEADROOM


# found by stepping each parameter until the facts asserted below hold
SPAN_WIDTH, SPAN_EXTRA_IN, SPAN_EXTRA_STEP = 25, 215, 1
CFIT_WIDTH, CFIT_EXTRA = 22, 217
CFIT_LEAVES = 13                      # string range leaves of the inside case; the outside case has one more
PFIT_WIDTHS = (50, 50, 50, 50, 50, 8, 1)
PFIT_IN = [0, 1, 2, 3, 4, 5]               # the outside case projects column 6 too
STAGE_WIDTHS_IN = (20, 23, 13)
STAGE_WIDTHS_OUT = (20, 23, 12)


# ---- tables ------------------------------------------------------------------------------------------------------------------
def _ob():
    import oceanbase_b200
    return oceanbase_b200


def _words(n, width, seed):
    """n distinct words of width to width + 4 bytes (lengths differ: a dictionary with variable-length entries)"""
    rng = np.random.default_rng(seed)
    return [b"w%05d" % i + bytes(rng.integers(97, 123, size=width - 6 + i % 5, dtype=np.uint8)) for i in range(n)]


@functools.lru_cache(maxsize=None)
def small_table(rpb, n_blocks, seed=1):
    """0 INT DICT 0..59, 1 VARCHAR DICT of 200 words, 2 INT RAW 0..99 (bit-packed, flat), 3 INT RAW with NULLs (not flat),
    4-6 INT DICT 0..29 / 0..39 / 0..49, 7 VARCHAR RAW of 40 to 80 bytes (projection span over the cap at 400 rows per block),
    8-13 INT RAW 0..99"""
    ob = _ob()
    n = rpb * n_blocks
    rng = np.random.default_rng(seed)
    words = _words(200, 12, seed)
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_DICT, rng.integers(0, 60, size=n, dtype=np.int64)),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, [words[i] for i in rng.integers(0, 200, size=n)]),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 100, size=n, dtype=np.int64)),
            ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(-1000, 1000, size=n, dtype=np.int64),
                      nulls=(rng.random(n) < 0.05).astype(np.uint8))]
    for hi in (30, 40, 50):
        cols.append(ob.Column(ob.OBJ_INT, ob.ENC_DICT, rng.integers(0, hi, size=n, dtype=np.int64)))
    cols.append(ob.Column(ob.OBJ_VARCHAR, ob.ENC_RAW, [bytes(rng.integers(97, 123, size=int(k), dtype=np.uint8))
                                                        for k in rng.integers(40, 81, size=n)]))
    for _ in range(6):
        cols.append(ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 100, size=n, dtype=np.int64)))
    return ob.encode_table(cols, rpb), tuple(words)


@functools.lru_cache(maxsize=None)
def dict_span_table(extra, width=SPAN_WIDTH, rpb=400, n_blocks=8):
    """0 VARCHAR DICT: every block holds the same 400 words (the first `extra` one byte longer) in its own order,
    so every block's region is the same; 1 INT RAW 0..99"""
    ob = _ob()
    words = [w + (b"+" if i < extra else b"") for i, w in enumerate(_words(400, width, 7))]
    rng = np.random.default_rng(extra)
    s = [words[i] for _ in range(n_blocks) for i in rng.permutation(rpb) % len(words)]
    cols = [ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s), ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 100, size=len(s), dtype=np.int64))]
    return ob.encode_table(cols, rpb), tuple(words)


@functools.lru_cache(maxsize=None)
def count_fit_table(extra, width=CFIT_WIDTH, rpb=400, n_blocks=8):
    """0 INT RAW 0..2^40 (41-bit), 1 VARCHAR DICT of the same 400 words in every block (`extra` of them one byte longer)"""
    ob = _ob()
    words = [w + (b"+" if i < extra else b"") for i, w in enumerate(_words(400, width, 9))]
    rng = np.random.default_rng(100 + extra)
    s = [words[i] for _ in range(n_blocks) for i in rng.permutation(rpb) % len(words)]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 1 << 40, size=len(s), dtype=np.int64)),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, s)]
    return ob.encode_table(cols, rpb), tuple(sorted(words))


@functools.lru_cache(maxsize=None)
def fixed_str_table(rpb, length, n_blocks=6):
    """0 VARCHAR of `length` bytes in every row (RAW, fixed length: one region of rows x length bytes), 1 INT RAW 0..99"""
    ob = _ob()
    rng = np.random.default_rng(length)
    n = rpb * n_blocks
    s = [bytes(r) for r in rng.integers(97, 123, size=(n, length), dtype=np.uint8)]
    cols = [ob.Column(ob.OBJ_VARCHAR, ob.ENC_RAW, s), ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 100, size=n, dtype=np.int64))]
    return ob.encode_table(cols, rpb), ()


@functools.lru_cache(maxsize=None)
def widths_table(widths, rpb, n_blocks=6, seed=3):
    """INT RAW columns bit-packed to the given widths (values 0 .. 2^w - 1, every width reached in every block)"""
    ob = _ob()
    rng = np.random.default_rng(seed)
    n = rpb * n_blocks
    cols = []
    for w in widths:
        v = rng.integers(0, 1 << w, size=n, dtype=np.int64)
        v[::rpb] = (1 << w) - 1
        cols.append(ob.Column(ob.OBJ_INT, ob.ENC_RAW, v))
    return ob.encode_table(cols, rpb), ()


@functools.lru_cache(maxsize=None)
def cs_table(rpb=400, n_blocks=10):
    """CS blocks: 0 CS_INTEGER 0..99, 1 CS_STRING of 5 to 30 bytes"""
    ob = _ob()
    rng = np.random.default_rng(5)
    n = rpb * n_blocks
    s = [b"c%d" % k + b"s" * int(k % 27) for k in rng.integers(0, 5000, size=n)]
    cols = [ob.Column(ob.OBJ_INT, ob.ENC_CS_INTEGER, rng.integers(0, 100, size=n, dtype=np.int64)),
            ob.Column(ob.OBJ_VARCHAR, ob.ENC_CS_STRING, s)]
    return ob.encode_table(cols, rpb), ()


@functools.lru_cache(maxsize=None)
def big_dict_table(rpb=20000, n_blocks=2):
    """0 VARCHAR DICT with a distinct word per row (20000-entry dictionaries), 1 INT RAW 0..511 (9 bits)"""
    ob = _ob()
    rng = np.random.default_rng(11)
    n = rpb * n_blocks
    words = [b"k%06d" % i for i in range(n)]
    cols = [ob.Column(ob.OBJ_VARCHAR, ob.ENC_DICT, words), ob.Column(ob.OBJ_INT, ob.ENC_RAW, rng.integers(0, 512, size=n, dtype=np.int64))]
    return ob.encode_table(cols, rpb), tuple(words)


TABLES = {
    "s400": lambda: small_table(400, 24),
    "s512": lambda: small_table(512, 10),
    "s513": lambda: small_table(513, 10),
    "s600": lambda: small_table(600, 16),
    "s1024": lambda: small_table(1024, 5),
    "s1025": lambda: small_table(1025, 5),
    "span_in": lambda: dict_span_table(SPAN_EXTRA_IN),
    "span_out": lambda: dict_span_table(SPAN_EXTRA_IN + SPAN_EXTRA_STEP),
    "cfit": lambda: count_fit_table(CFIT_EXTRA),
    "pspan_in": lambda: fixed_str_table(409, 40),
    "pspan_out": lambda: fixed_str_table(512, 32),
    "pfit": lambda: widths_table(PFIT_WIDTHS, 400),
    "stage_in": lambda: widths_table(STAGE_WIDTHS_IN, 600),
    "stage_out": lambda: widths_table(STAGE_WIDTHS_OUT, 600),
    "no_stage": lambda: widths_table((60, 60, 60, 60), 8000, n_blocks=3),
    "cs": lambda: cs_table(),
    "big_dict": lambda: big_dict_table(),
}

@functools.lru_cache(maxsize=None)
def facts(name):
    table, _ = TABLES[name]()
    return table_facts(table, _u(table.block(0), 8, 4) >> 16)


# ---- cases -------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    table: str
    filter: Optional[Callable]            # (ob, words) -> filter expression
    proj: Sequence[int]
    expect: Tuple[int, int, int]          # (count kernel, projection kernel, projection flags)
    row_ids: bool = True
    cap: object = 0                       # max_selected_rows, or "sixteenth" / "sixteenth+1" of the table's rows
    knobs: dict = field(default_factory=dict)
    bitmap: bool = False                  # scan_bitmap with the rows the filter selects
    overflow: bool = False                # more rows pass than cap: the scan reports OB_BUF_NOT_ENOUGH

    def max_selected(self, total_rows):
        return {"sixteenth": total_rows // 16, "sixteenth+1": total_rows // 16 + 1}.get(self.cap, self.cap)


def W(col, op, *params):
    ob = _ob()
    return ob.White(col, getattr(ob, "WHITE_OP_" + op), tuple(params))


def AND(*c):
    return _ob().And(list(c))


def OR(*c):
    return _ob().Or(list(c))


# filters of small_table, each selecting well under 1/16 of the rows (the sparse split takes them)
F_PLANS = lambda ob, w: W(2, "LT", 5)                                                   # RAW integer: decode plans
F_CTA = lambda ob, w: AND(OR(W(2, "LT", 3), W(2, "GT", 97)), W(0, "LT", 59))              # nested: the generic tree
F_RECORDS = lambda ob, w: AND(W(0, "LT", 30), W(4, "LT", 29), W(5, "LT", 39), W(6, "LT", 49),
                              W(1, "IN", *w[:10]))                                      # 5 dictionary columns
F_CODED = lambda ob, w: AND(W(0, "LT", 3), W(4, "GE", 1))                                 # 2 dictionary columns
F_CODED4 = lambda ob, w: AND(W(0, "LT", 30), W(4, "LT", 15), W(5, "LT", 20), W(1, "IN", *w[:10]))
COUNTS = {NONE: None, BITMAP: F_PLANS, CTA: F_CTA, PLANS: F_PLANS, RECORDS: F_RECORDS, CODED: F_CODED}
PROJS = {P_NONE: ([], False), P_CTA: ([7, 2], True), P_SPARSE: ([7, 2], True), P_PLANS: ([3, 2], True),
         P_RECORDS: ([2, 0, 1], True)}


COUNT_NAMES = {NONE: "none", PLANS: "plans", RECORDS: "records", CODED: "coded", CTA: "cta", BITMAP: "bitmap"}
PROJ_NAMES = {P_NONE: "none", P_CTA: "cta", P_SPARSE: "sparse", P_PLANS: "plans", P_RECORDS: "records"}


def _pair_cases():
    out = []
    for cnt, flt in COUNTS.items():
        for pj, (proj, rid) in PROJS.items():
            if cnt == NONE and pj == P_SPARSE:
                continue                  # no filter selects nothing away: never the sparse split
            flags = {P_CTA: F_COMPACT, P_SPARSE: F_SPARSE | F_COMPACT}.get(pj, 0)
            out.append(Case(f"pair_{COUNT_NAMES[cnt]}_{PROJ_NAMES[pj]}", "s400", flt, proj, (cnt, pj, flags), row_ids=rid,
                            cap="sixteenth" if pj == P_SPARSE else 0, bitmap=cnt == BITMAP))
    return out


NF8 = [2, 3, 8, 9, 10, 11, 12, 13]
CASES = [
    # pipeline threshold: max_rows <= 512
    Case("pipe_512", "s512", lambda ob, w: AND(W(2, "LT", 50), W(8, "GE", 10)), [2, 9], (PLANS, P_RECORDS, 0)),
    Case("pipe_513", "s513", lambda ob, w: AND(W(2, "LT", 50), W(8, "GE", 10)), [2, 9], (CTA, P_CTA, F_COMPACT)),
    # filter shape
    Case("shape_and", "s400", lambda ob, w: AND(W(2, "LT", 50), W(8, "GE", 10)), [2], (PLANS, P_RECORDS, 0)),
    Case("shape_or", "s400", lambda ob, w: OR(W(2, "LT", 10), W(8, "GE", 90)), [2], (PLANS, P_RECORDS, 0)),
    Case("shape_nested", "s400", F_CTA, [2], (CTA, P_RECORDS, 0)),
    # filter columns: nf <= 8
    Case("nf_8", "s400", lambda ob, w: AND(*[W(c, "GE", 1) for c in NF8]), [2], (PLANS, P_RECORDS, 0)),
    Case("nf_9", "s400", lambda ob, w: AND(*[W(c, "GE", 1) for c in NF8], W(0, "GE", 1)), [2], (CTA, P_RECORDS, 0)),
    # count region span: 12288 bytes
    Case("count_span_cap", "span_in", lambda ob, w: W(0, "IN", *w[:3]), [1], (CODED, P_RECORDS, 0)),
    Case("count_span_over", "span_out", lambda ob, w: W(0, "IN", *w[:3]), [1], (CTA, P_RECORDS, 0)),
    Case("count_cs_string", "cs", lambda ob, w: W(1, "GT", b"c3"), [], (CTA, P_RECORDS, 0)),
    # records for counting: max_rows <= 1024 (past the natural pipeline threshold: OBGPU_PIPE=1)
    Case("rec_1024", "s1024", lambda ob, w: W(0, "LT", 30), [2], (CODED, P_RECORDS, 0), knobs={"OBGPU_PIPE": "1"}),
    Case("rec_1025", "s1025", lambda ob, w: W(0, "LT", 30), [2], (PLANS, P_RECORDS, 0), knobs={"OBGPU_PIPE": "1"}),
    Case("string_range_plans", "s400", lambda ob, w: W(1, "GT", w[100]), [2], (PLANS, P_RECORDS, 0)),
    # batch codes: the first four filter columns
    Case("codes_four", "s400", F_CODED4, [2], (CODED, P_RECORDS, 0)),
    Case("codes_fifth", "s400", F_RECORDS, [2], (RECORDS, P_RECORDS, 0)),
    Case("codes_off", "s400", F_CODED4, [2], (RECORDS, P_RECORDS, 0), knobs={"OBGPU_STR_CODES": "0"}),
    # two CTAs per SM, count
    Case("count_fit_in", "cfit", lambda ob, w: AND(W(0, "GE", 0), *[W(1, "GT", w[i]) for i in range(CFIT_LEAVES)]), [0],
         (PLANS, P_RECORDS, 0)),
    Case("count_fit_out", "cfit", lambda ob, w: AND(W(0, "GE", 0), *[W(1, "GT", w[i]) for i in range(CFIT_LEAVES + 1)]), [0],
         (CTA, P_RECORDS, 0)),
    # projection span: 16384 bytes
    Case("proj_span_cap", "pspan_in", None, [0], (NONE, P_PLANS, 0)),
    Case("proj_span_over", "pspan_out", None, [0], (NONE, P_CTA, 0)),
    # records or plans for projection
    Case("proj_records", "s400", F_PLANS, [2, 0], (PLANS, P_RECORDS, 0)),
    Case("proj_plans", "s400", F_PLANS, [2, 3], (PLANS, P_PLANS, 0)),
    # two CTAs per SM, projection
    Case("proj_fit_in", "pfit", None, PFIT_IN, (NONE, P_RECORDS, 0)),
    Case("proj_fit_out", "pfit", None, PFIT_IN + [6], (NONE, P_CTA, 0)),
    # sparse split: max_selected_rows * 16 <= total rows
    Case("sparse_at", "s600", F_PLANS, [2, 0], (CTA, P_SPARSE, F_SPARSE | F_COMPACT), cap="sixteenth"),
    Case("sparse_over", "s600", F_PLANS, [2, 0], (CTA, P_CTA, F_COMPACT), cap="sixteenth+1"),
    Case("sparse_no_filter", "s600", None, [2, 0], (NONE, P_CTA, F_COMPACT), cap="sixteenth", overflow=True),
    # staging of obgpu_project_kernel
    Case("stage_compact", "stage_in", None, [0, 1], (NONE, P_CTA, F_COMPACT)),
    Case("stage_block", "stage_out", None, [0, 1], (NONE, P_CTA, 0)),
    Case("no_stage", "no_stage", lambda ob, w: W(0, "LT", 1 << 58), [0, 1, 2, 3], (CTA, P_CTA, F_NO_STAGE)),
    # row ids alone still take a projection kernel
    Case("row_ids_pipe", "s400", F_PLANS, [], (PLANS, P_RECORDS, 0)),
    Case("row_ids_cta", "s600", F_PLANS, [], (CTA, P_CTA, 0)),
] + _pair_cases()
CASE = {c.name: c for c in CASES}

# a filter whose obgpu_count_kernel working set exceeds shared memory: 15 leaves, 14 of them with a predicate bitset over a
# 20000-entry dictionary, and a 9-bit column staged next to them
BIG_FILTER = lambda ob, w: AND(W(1, "GE", 0), *[W(0, "NE", w[i]) for i in range(14)])


# ---- the facts ---------------------------------------------------------------------------------------------------------------
def test_row_counts():
    for name, rows in (("s400", 400), ("s512", 512), ("s513", 513), ("s600", 600), ("s1024", 1024), ("s1025", 1025)):
        assert facts(name).max_rows == rows, name
    assert facts("s600").total_rows % 16 == 0


def test_small_table_columns():
    f = facts("s400")
    assert all(f.span[c] <= COUNT_SPAN_CAP for c in NF8 + [0, 1])
    assert f.pspan[7] > PROJ_SPAN_CAP                      # projecting column 7 leaves the pipelined kernel
    assert all(f.max_dict[c] > 0 for c in (0, 1, 4, 5, 6)) and all(f.max_dict[c] == 0 for c in (2, 3, 7))


def test_count_span_pair():
    assert facts("span_in").span[0] == COUNT_SPAN_CAP
    assert facts("span_out").span[0] == COUNT_SPAN_CAP + 16


def test_proj_span_pair():
    assert facts("pspan_in").pspan[0] == PROJ_SPAN_CAP
    assert facts("pspan_out").pspan[0] == PROJ_SPAN_CAP + 16
    assert not compact(facts("pspan_out"), [0])


def test_count_fit_pair():
    f = facts("cfit")
    assert f.span[1] <= COUNT_SPAN_CAP
    inside, outside = count_pipe_bytes(f, [0, 1], CFIT_LEAVES), count_pipe_bytes(f, [0, 1], CFIT_LEAVES + 1)
    assert two_ctas(inside, H100_MAX_SMEM) and not two_ctas(outside, H100_MAX_SMEM), (inside, outside)
    assert count_cta_bytes(f, [0, 1], CFIT_LEAVES + 1) * WARPS <= H100_MAX_SMEM


def test_proj_fit_pair():
    f = facts("pfit")
    inside, outside = proj_pipe_bytes(f, PFIT_IN, True), proj_pipe_bytes(f, PFIT_IN + [6], True)
    assert two_ctas(inside, H100_MAX_SMEM) and not two_ctas(outside, H100_MAX_SMEM), (inside, outside)
    assert all(f.pspan[c] <= PROJ_SPAN_CAP for c in range(7))


def test_sparse_pair_selects_under_the_cap():
    table, words = TABLES["s600"]()
    want = ora.scan_table(table, F_PLANS(None, words), [], [], [])
    assert want["selected"] <= table.total_rows // 16
    table, words = TABLES["s400"]()
    for flt in (F_PLANS, F_CTA, F_RECORDS, F_CODED):
        assert ora.scan_table(table, flt(None, words), [], [], [])["selected"] <= table.total_rows // 16


def test_staging_pair():
    f_in, f_out = facts("stage_in"), facts("stage_out")
    s_in, s_out = f_in.span[0] + f_in.span[1], f_out.span[0] + f_out.span[1]
    assert s_in == s_out and s_in * 4 == f_in.block_bytes * 3
    assert s_out * 4 > f_out.block_bytes * 3


def test_no_stage_blocks_exceed_shared_memory():
    assert facts("no_stage").block_bytes > H100_MAX_SMEM
    assert not compact(facts("no_stage"), [0, 1, 2, 3])


def test_cs_string_has_no_region():
    assert facts("cs").span[1] is None


def test_big_filter_working_set():
    f = facts("big_dict")
    assert f.max_dict[0] == 20002 and f.span[1] <= 24576 and f.span[0] > 24576
    assert count_cta_bytes(f, [1, 0], 14) * WARPS > H100_MAX_SMEM


def test_expected_compact_flags():
    for c in CASES:
        if c.expect[1] in (P_CTA, P_SPARSE) and not c.expect[2] & F_NO_STAGE:
            assert bool(c.expect[2] & F_COMPACT) == compact(facts(c.table), list(c.proj)), c.name
