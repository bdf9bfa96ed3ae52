"""Host-side mirror of the scan operator surface over the C-ABI.

Names follow the reference: a *white filter* is sql::ObWhiteFilterExecutor (one column, one
ObWhiteFilterOperatorType, constants); And / Or are the logic nodes of the
ObPushdownFilterExecutor tree (sql/engine/basic/ob_pushdown_filter.h:690-934); a PageBatch is what
ObSSTableRowScanner feeds block by block to ObIMicroBlockReader::init; ScanResult holds what
ObMicroBlockDecoder::get_rows would have written into the ObExpr vectors, dense over the batch.
"""
import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Union

import numpy as np

from . import capi
from .capi import lib, check


# common::ObDatum: 8-byte pointer + {len:29, flag:2, null:1}, 12 packed bytes (share/datum/ob_datum.h:109-177)
DATUM_DTYPE = np.dtype([("ptr", "<u8"), ("pack", "<u4")], align=False)
DATUM_NULL_BIT = 0x80000000


# ---- filter tree ---------------------------------------------------------------------------------
@dataclass
class White:
    col: int
    op: int
    params: Sequence = ()     # ints, bytes, or None (NULL constant)


@dataclass
class And:
    children: Sequence


@dataclass
class Or:
    children: Sequence


FilterExpr = Union[White, And, Or]


def flatten_filter(expr: Optional[FilterExpr], node_cls=capi.FilterNode, param_cls=capi.FilterParam,
                   filter_cls=capi.Filter):
    """Post-order flattening (root last). Returns (filter_struct, keepalive) or (None, None)."""
    if expr is None:
        return None, None
    nodes, params, keep = [], [], []

    def visit(e):
        if isinstance(e, White):
            nd = node_cls()
            nd.kind, nd.op, nd.col = capi.NODE_WHITE, e.op, e.col
            nd.param_begin, nd.n_params, nd.n_children = len(params), len(e.params), 0
            for v in e.params:
                p = param_cls()
                if v is None:
                    p.is_null = 1
                elif isinstance(v, (bytes, bytearray)):
                    b = bytes(v)
                    keep.append(b)
                    p.ptr, p.len = b, len(b)
                else:
                    iv = int(v)
                    if iv >= 1 << 63:
                        iv -= 1 << 64
                    p.i64 = iv
                params.append(p)
            nodes.append(nd)
        else:
            for c in e.children:
                visit(c)
            nd = node_cls()
            nd.kind = capi.NODE_AND if isinstance(e, And) else capi.NODE_OR
            nd.n_children = len(e.children)
            nodes.append(nd)

    visit(expr)
    node_arr = (node_cls * len(nodes))(*nodes)
    param_arr = (param_cls * max(len(params), 1))(*params)
    f = filter_cls()
    f.nodes, f.n_nodes = node_arr, len(nodes)
    f.params, f.n_params = param_arr, len(params)
    return f, (node_arr, param_arr, keep)


def group_tuples(keys, nulls, heap, n, types):
    """Groups in obgpu_result_fetch_group_columns' host layout -> one tuple per group: per column (obj_type, datum_len) of
    types, a Python int in the column's value domain (unsigned types non-negative), bytes, or None for NULL."""
    heap_b = heap.tobytes()
    per_col = []
    for c, (obj_type, dlen) in enumerate(types):
        k = keys[c].tolist()
        if dlen == 0:
            vals = [heap_b[k[g]:k[g + 1]] for g in range(n)]
        elif obj_type in (capi.OBJ_UINT64, capi.OBJ_UINT32, capi.OBJ_UTINYINT, capi.OBJ_USMALLINT, capi.OBJ_UMEDIUMINT, capi.OBJ_YEAR):
            vals = [v & ((1 << 64) - 1) for v in k[:n]]
        else:
            vals = k[:n]
        per_col.append([None if z else v for v, z in zip(vals, nulls[c, :n].tolist())])
    return list(zip(*per_col)) if n else []


def sort_keys(keys):
    """sort keys (a store column, or (col, desc, nulls_first)) -> the int32 [n][3] array of obgpu_sort_key"""
    ks = [(kk, 0, 0) if isinstance(kk, int) else tuple(int(x) for x in kk) for kk in keys]
    return np.array(ks, dtype=np.int32).reshape(-1, 3)


def fetch_top_rows(fetch, n, heap_bytes, types):
    """rows in obgpu_result_fetch_top_rows' layout (fetch(blocks, rows, vals, nulls, heap) fills it) -> (positions, rows) as
    ScanResult.top_rows returns them; types: (obj_type, datum_len) per output column"""
    no = len(types)
    blocks, rows = np.zeros(max(n, 1), dtype=np.int32), np.zeros(max(n, 1), dtype=np.int32)
    vals = np.zeros((no, n + 1), dtype=np.int64)
    nulls = np.zeros((no, max(n, 1)), dtype=np.uint8)
    heap = np.zeros(max(heap_bytes, 1), dtype=np.uint8)
    fetch(blocks.ctypes.data, rows.ctypes.data, vals.ctypes.data, nulls.ctypes.data, heap.ctypes.data)
    positions = list(zip(blocks[:n].tolist(), rows[:n].tolist()))
    return positions, (group_tuples(vals, nulls, heap, n, types) if no else [()] * n)


# ---- context / batch / result ----------------------------------------------------------------------
class ScanContext:
    """obgpu_ctx: one per worker thread (device + stream)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self._h = C.c_void_p()
        code = lib.obgpu_ctx_create(device, C.byref(self._h))
        if code != capi.OB_SUCCESS:
            raise capi.ObGpuError(code, "obgpu_ctx_create", "no usable CUDA device; there is no CPU fallback")
        self.device = device
        if stream is not None:
            self.set_stream(stream)

    def set_stream(self, cuda_stream_ptr: Optional[int]):
        check(lib.obgpu_ctx_set_stream(self._h, C.c_void_p(cuda_stream_ptr or 0)), "obgpu_ctx_set_stream", self._h)

    def synchronize(self):
        check(lib.obgpu_ctx_synchronize(self._h), "obgpu_ctx_synchronize", self._h)

    @property
    def launch_count(self) -> int:
        return lib.obgpu_ctx_launch_count(self._h)

    def set_profiling(self, enable: bool = True):
        check(lib.obgpu_ctx_set_profiling(self._h, 1 if enable else 0), "obgpu_ctx_set_profiling", self._h)

    def kernel_times_ms(self, last_n: int = 256) -> np.ndarray:
        ms = np.zeros(max(last_n, 1), dtype=np.float32)
        n = C.c_int32(0)
        check(lib.obgpu_ctx_kernel_times(self._h, ms.ctypes.data, last_n, C.byref(n)), "obgpu_ctx_kernel_times",
              self._h)
        return ms[:n.value].copy()

    def last_error(self) -> str:
        return (lib.obgpu_ctx_last_error(self._h) or b"").decode()

    def last_plan(self):
        """(count kernel, projection kernel, projection flags) the last scan on this ctx chose: obgpu_ctx_scan_plan, numbered
        as OBGPU_SCAN_COUNT_* / OBGPU_SCAN_PROJ_* / OBGPU_SCAN_PROJ_FLAG_* in include/obgpu_scan.h."""
        cnt, proj, flags = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        check(lib.obgpu_ctx_scan_plan(self._h, C.byref(cnt), C.byref(proj), C.byref(flags)), "obgpu_ctx_scan_plan", self._h)
        return cnt.value, proj.value, flags.value

    def group_accumulator(self, n_group_cols: int, aggs) -> "GroupAccumulator":
        """obgpu_groups on this ctx: merges the groups of ScanResult.group_by_columns / group_by_values of several results by value."""
        return GroupAccumulator.create(self, n_group_cols, aggs)

    def open_batch(self, table, device_image_ptr: Optional[int] = None, host_view: bool = True,
                   image_size: Optional[int] = None, compressor: Optional[int] = None) -> "PageBatch":
        return PageBatch(self, table, device_image_ptr, host_view, image_size, compressor)

    def bitmap_to_row_ids(self, bitmap: np.ndarray, start: int, to: int, limit: int, id_offset: int = 0):
        """common::ObBitmap::get_row_ids. Returns (row_ids, next_from)."""
        bm = np.ascontiguousarray(bitmap, dtype=np.uint8)
        out = np.zeros(max(min(limit, max(to - start, 0)), 1), dtype=np.int32)
        frm, cnt = C.c_int64(start), C.c_int64(0)
        check(lib.obgpu_bitmap_to_row_ids(self._h, bm.ctypes.data, bm.size, C.byref(frm), to, limit, id_offset,
                                          out.ctypes.data, C.byref(cnt)), "obgpu_bitmap_to_row_ids", self._h)
        return out[:cnt.value].copy(), frm.value

    def close(self):
        if self._h:
            lib.obgpu_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PageBatch:
    """obgpu_batch: N micro-blocks resident in HBM."""

    def __init__(self, ctx: ScanContext, table, device_image_ptr: Optional[int] = None, host_view: bool = True,
                 image_size: Optional[int] = None, compressor: Optional[int] = None):
        """host_view=False: a device-resident image is opened without a host copy of it (table.image may then be
        None; the headers are surveyed on the device).
        compressor (capi.COMPRESSOR_*): the blocks of `table` are in stored form (sstable.compress_table) and are decoded on
        the device by obgpu_batch_open_compressed into an image the batch owns (device_image()): LZ4 / LZ4_1_9_1 (LZ4
        blocks), ZLIB (zlib streams) or ZSTD_1_3_8 (zstd frames); None: plain blocks."""
        self.ctx = ctx
        self.table = table
        self._h = C.c_void_p()
        img = table.image
        offs = np.ascontiguousarray(table.offsets, dtype=np.int64)
        sizes = np.ascontiguousarray(table.sizes, dtype=np.int64)
        if compressor is not None:
            if device_image_ptr is None:
                img = np.ascontiguousarray(img, dtype=np.uint8)
                code = lib.obgpu_batch_open_compressed(ctx._h, img.ctypes.data, img.size, offs.ctypes.data, sizes.ctypes.data,
                                                       len(offs), 0, int(compressor), C.byref(self._h))
            else:
                size = int(image_size) if image_size is not None else img.size
                code = lib.obgpu_batch_open_compressed(ctx._h, C.c_void_p(device_image_ptr), size, offs.ctypes.data,
                                                       sizes.ctypes.data, len(offs), 1, int(compressor), C.byref(self._h))
            check(code, "obgpu_batch_open_compressed", ctx._h)
        elif device_image_ptr is None:
            code = lib.obgpu_batch_open(ctx._h, img.ctypes.data, img.size, offs.ctypes.data, sizes.ctypes.data,
                                        len(offs), 0, None, C.byref(self._h))
        else:
            size = int(image_size) if image_size is not None else img.size
            code = lib.obgpu_batch_open(ctx._h, C.c_void_p(device_image_ptr), size, offs.ctypes.data,
                                        sizes.ctypes.data, len(offs), 1,
                                        img.ctypes.data if (host_view and img is not None) else None, C.byref(self._h))
        if compressor is None:
            check(code, "obgpu_batch_open", ctx._h)
        self.n_blocks = len(offs)
        tr = C.c_int64(0)
        check(lib.obgpu_batch_total_rows(self._h, C.byref(tr)), "obgpu_batch_total_rows", ctx._h)
        self.total_rows = tr.value

    @classmethod
    def from_macro_blocks(cls, ctx: "ScanContext", macro_image, macro_block_size: int, n_macro: int, device_ptr: Optional[int] = None,
                          table=None) -> "PageBatch":
        """obgpu_batch_open_macro_blocks: disk-format macro blocks (sstable.build_macro_blocks) parsed and re-laid on the device.
        macro_image: host uint8 array, or None with device_ptr naming a device-resident copy of n_macro * macro_block_size bytes."""
        self = cls.__new__(cls)
        self.ctx = ctx
        self.table = table
        self._h = C.c_void_p()
        n_micro = C.c_int32(0)
        size = n_macro * macro_block_size
        if device_ptr is None:
            img = np.ascontiguousarray(macro_image, dtype=np.uint8)
            code = lib.obgpu_batch_open_macro_blocks(ctx._h, img.ctypes.data, size, macro_block_size, n_macro, 0, C.byref(self._h), C.byref(n_micro))
        else:
            code = lib.obgpu_batch_open_macro_blocks(ctx._h, C.c_void_p(device_ptr), size, macro_block_size, n_macro, 1, C.byref(self._h),
                                                     C.byref(n_micro))
        check(code, "obgpu_batch_open_macro_blocks", ctx._h)
        self.n_blocks = n_micro.value
        tr = C.c_int64(0)
        check(lib.obgpu_batch_total_rows(self._h, C.byref(tr)), "obgpu_batch_total_rows", ctx._h)
        self.total_rows = tr.value
        return self

    def device_image(self):
        """(device address, bytes) of the image the batch's blocks live in (obgpu_batch_device_image). For a batch that owns
        its image (host image, macro blocks, compressed blocks) scan(string_base=device_image()[0]) yields device addresses."""
        p, n = C.c_void_p(), C.c_int64(0)
        check(lib.obgpu_batch_device_image(self._h, C.byref(p), C.byref(n)), "obgpu_batch_device_image", self.ctx._h)
        return p.value or 0, n.value

    def block_info(self, i):
        rc, cc = C.c_int64(0), C.c_int32(0)
        check(lib.obgpu_batch_block_info(self._h, i, C.byref(rc), C.byref(cc)), "obgpu_batch_block_info", self.ctx._h)
        return rc.value, cc.value

    def scan(self, filter: Optional[FilterExpr], proj_cols: Sequence[int], want_row_ids=False, string_base=0,
             max_selected_rows=0) -> "ScanResult":
        f, keep = flatten_filter(filter)
        proj = (C.c_int32 * max(len(proj_cols), 1))(*proj_cols)
        spec = capi.ScanSpec()
        spec.filter = C.pointer(f) if f is not None else None
        spec.proj_cols, spec.n_proj = proj, len(proj_cols)
        spec.want_row_ids = 1 if want_row_ids else 0
        spec.string_base = string_base
        spec.max_selected_rows = max_selected_rows
        h = C.c_void_p()
        check(lib.obgpu_scan(self._h, C.byref(spec), C.byref(h)), "obgpu_scan", self.ctx._h)
        return ScanResult(self, h, len(proj_cols))

    def scan_bitmap(self, bitmap: "CGBitmap", proj_cols: Sequence[int], row_offset: int = 0, want_row_ids=False, string_base=0,
                    max_selected_rows=0) -> "ScanResult":
        """obgpu_scan_bitmap: project the rows a range bitmap selects (ObCGRowScanner::get_next_rows(count, capacity, bitmap))."""
        proj = (C.c_int32 * max(len(proj_cols), 1))(*proj_cols)
        spec = capi.ScanSpec()
        spec.filter = None
        spec.proj_cols, spec.n_proj = proj, len(proj_cols)
        spec.want_row_ids = 1 if want_row_ids else 0
        spec.string_base = string_base
        spec.max_selected_rows = max_selected_rows
        h = C.c_void_p()
        check(lib.obgpu_scan_bitmap(self._h, bitmap._h, row_offset, C.byref(spec), C.byref(h)), "obgpu_scan_bitmap", self.ctx._h)
        return ScanResult(self, h, len(proj_cols))

    # ---- skip index (include/obgpu_skip_index.h) ---------------------------------------------------
    def set_agg_rows(self, agg_rows: Optional[np.ndarray], agg_off: Optional[np.ndarray] = None):
        """Attach the blocks' serialized aggregate rows (block b: agg_rows[agg_off[b]:agg_off[b + 1]]); None detaches.
        Scans of this batch then prune with them."""
        if agg_rows is None:
            check(lib.obgpu_batch_set_agg_rows(self._h, None, None), "obgpu_batch_set_agg_rows", self.ctx._h)
            return
        rows = np.ascontiguousarray(agg_rows, dtype=np.uint8)
        off = np.ascontiguousarray(agg_off, dtype=np.int64)
        assert len(off) == self.n_blocks + 1
        check(lib.obgpu_batch_set_agg_rows(self._h, rows.ctypes.data, off.ctypes.data), "obgpu_batch_set_agg_rows",
              self.ctx._h)

    def skip_index_filter(self, expr: FilterExpr) -> np.ndarray:
        """ObSSTableIndexFilter::check_range per block: uint8 verdicts (capi.BOOL_MASK_*)."""
        f, keep = flatten_filter(expr)
        out = np.zeros(max(self.n_blocks, 1), dtype=np.uint8)
        check(lib.obgpu_batch_skip_index_filter(self._h, C.byref(f), out.ctypes.data), "obgpu_batch_skip_index_filter",
              self.ctx._h)
        return out[:self.n_blocks]

    # ---- reference-granularity calls -------------------------------------------------------------
    def filter_white(self, block, col, op, params=(), start=0, count=None) -> np.ndarray:
        f, keep = flatten_filter(White(col, op, params))
        return self.filter_tree(block, None, start, count, _flat=f)

    def filter_tree(self, block, expr, start=0, count=None, _flat=None) -> np.ndarray:
        f = _flat
        if f is None:
            f, keep = flatten_filter(expr)
        if count is None:
            count = self.block_info(block)[0] - start
        out = np.zeros(max(count, 1), dtype=np.uint8)
        check(lib.obgpu_filter_tree(self._h, block, C.byref(f), start, count, out.ctypes.data), "obgpu_filter_tree",
              self.ctx._h)
        return out[:count]

    def project_fixed(self, block, col, row_ids, elem_len=8, vec_offset=0, data=None, nulls=None):
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        total = vec_offset + len(rid)
        if data is None:
            data = np.zeros(total * elem_len, dtype=np.uint8)
        if nulls is None:
            nulls = np.zeros((total + 63) // 64, dtype=np.uint64)
        hn = C.c_int32(0)
        check(lib.obgpu_project_fixed(self._h, block, col, rid.ctypes.data, len(rid), vec_offset, data.ctypes.data,
                                      elem_len, nulls.ctypes.data, C.byref(hn)), "obgpu_project_fixed", self.ctx._h)
        return data, nulls, hn.value

    def project_discrete(self, block, col, row_ids, string_base=0, vec_offset=0):
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        total = vec_offset + len(rid)
        ptrs = np.zeros(total, dtype=np.uint64)
        lens = np.zeros(total, dtype=np.int32)
        nulls = np.zeros((total + 63) // 64, dtype=np.uint64)
        hn = C.c_int32(0)
        check(lib.obgpu_project_discrete(self._h, block, col, rid.ctypes.data, len(rid), vec_offset, string_base,
                                         ptrs.ctypes.data, lens.ctypes.data, nulls.ctypes.data, C.byref(hn)),
              "obgpu_project_discrete", self.ctx._h)
        return ptrs, lens, nulls, hn.value

    def project_datums(self, block, col, row_ids, datums: np.ndarray, datum_offset=0, string_base=0):
        """ObMicroBlockDecoder::get_rows, datum format: fills `datums` (structured array DATUM_DTYPE, 12 bytes each) from
        datum_offset on. Integer datums must already point at their 8-byte slots."""
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        check(lib.obgpu_project_datums(self._h, block, col, rid.ctypes.data, len(rid), datum_offset, string_base,
                                       datums.ctypes.data), "obgpu_project_datums", self.ctx._h)
        return datums

    # ---- string cells as bytes (columns whose values the device rebuilt: HEX_PACKING / STRING_DIFF / STRING_PREFIX) ----
    def column_materialised(self, col) -> bool:
        m = C.c_int32(0)
        check(lib.obgpu_batch_column_materialised(self._h, col, C.byref(m)), "obgpu_batch_column_materialised", self.ctx._h)
        return bool(m.value)

    def project_strings(self, block, col, row_ids):
        """obgpu_project_strings: (heap uint8, offsets int64 [n + 1], nulls words) of the listed rows of one block."""
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        n = len(rid)
        off = np.zeros(n + 1, dtype=np.int64)
        nulls = np.zeros(max((n + 63) // 64, 1), dtype=np.uint64)
        need, hn = C.c_int64(0), C.c_int32(0)
        heap = np.zeros(1, dtype=np.uint8)
        rc = lib.obgpu_project_strings(self._h, block, col, rid.ctypes.data, n, heap.ctypes.data, 0, off.ctypes.data, nulls.ctypes.data,
                                       C.byref(hn), C.byref(need))
        if rc == capi.OB_BUF_NOT_ENOUGH:
            heap = np.zeros(max(need.value, 1), dtype=np.uint8)
            rc = lib.obgpu_project_strings(self._h, block, col, rid.ctypes.data, n, heap.ctypes.data, heap.size, off.ctypes.data,
                                           nulls.ctypes.data, C.byref(hn), C.byref(need))
        check(rc, "obgpu_project_strings", self.ctx._h)
        return heap[:need.value], off, nulls

    # ---- dictionary surface (pushdown GROUP BY, black filter on one dictionary column) ----
    def distinct_count(self, block, col) -> int:
        """ObIMicroBlockReader::get_distinct_count."""
        n = C.c_int64(0)
        check(lib.obgpu_block_distinct_count(self._h, block, col, C.byref(n)), "obgpu_block_distinct_count", self.ctx._h)
        return n.value

    def read_distinct(self, block, col, string_base=0):
        """ObIMicroBlockReader::read_distinct: (vals uint64, lens int32) in dictionary order; strings: vals are addresses
        string_base + offset in the caller's image."""
        n = self.distinct_count(block, col)
        vals = np.zeros(max(n, 1), dtype=np.uint64)
        lens = np.zeros(max(n, 1), dtype=np.int32)
        got = C.c_int64(0)
        check(lib.obgpu_block_read_distinct(self._h, block, col, string_base, vals.ctypes.data, lens.ctypes.data, n, C.byref(got)),
              "obgpu_block_read_distinct", self.ctx._h)
        return vals[:n], lens[:n]

    def read_reference(self, block, col, row_ids) -> np.ndarray:
        """ObIMicroBlockReader::read_reference: ref per listed row, the distinct count for NULL rows."""
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        refs = np.zeros(max(len(rid), 1), dtype=np.uint32)
        check(lib.obgpu_block_read_reference(self._h, block, col, rid.ctypes.data, len(rid), refs.ctypes.data),
              "obgpu_block_read_reference", self.ctx._h)
        return refs[:len(rid)]

    def filter_dict_pass(self, block, col, entry_pass, null_pass=False, start=0, count=None) -> np.ndarray:
        """Black filter on one dictionary column: verdict per distinct value -> ObBitmap bytes of rows [start, start + count)."""
        ep = np.ascontiguousarray(entry_pass, dtype=np.uint8)
        if count is None:
            count = self.block_info(block)[0] - start
        out = np.zeros(max(count, 1), dtype=np.uint8)
        check(lib.obgpu_filter_dict_pass(self._h, block, col, ep.ctypes.data if len(ep) else None, len(ep), int(bool(null_pass)),
                                         start, count, out.ctypes.data), "obgpu_filter_dict_pass", self.ctx._h)
        return out[:count]

    def group_by(self, block, group_col, aggs, row_ids):
        """Pushdown GROUP BY on one block: aggs = [(kind, store col or -1)]; returns int64 [n_aggs][groups][2]
        (groups = distinct count + 1, the last one is the NULL group)."""
        rid = np.ascontiguousarray(row_ids, dtype=np.int32)
        g = self.distinct_count(block, group_col) + 1
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        out = np.zeros((len(aggs), g, 2), dtype=np.int64)
        n = C.c_int64(0)
        check(lib.obgpu_block_group_by(self._h, block, group_col, spec.ctypes.data, len(aggs), rid.ctypes.data, len(rid),
                                       out.ctypes.data, g, C.byref(n)), "obgpu_block_group_by", self.ctx._h)
        assert n.value == g
        return out

    def close(self):
        if self._h:
            if self.ctx._h:  # the C ctx owns the stream: never touch a batch after its ctx is gone
                lib.obgpu_batch_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CGBitmap:
    """obgpu_cg_bitmap: ObCGBitmap of a row range, device resident (column-store tables: filters of different column groups meet here)."""

    def __init__(self, ctx: "ScanContext", n_rows: int, all_true: bool = False):
        self.ctx, self.n_rows = ctx, n_rows
        self._h = C.c_void_p()
        check(lib.obgpu_cg_bitmap_create(ctx._h, n_rows, 1 if all_true else 0, C.byref(self._h)), "obgpu_cg_bitmap_create", ctx._h)

    def apply(self, result: "ScanResult", row_offset: int = 0, op: str = "and"):
        code = {"set": 0, "and": 1, "or": 2}[op]
        check(lib.obgpu_cg_bitmap_apply_result(self._h, result._h, row_offset, code), "obgpu_cg_bitmap_apply_result", self.ctx._h)

    def popcnt(self, lo: int = 0, hi: Optional[int] = None) -> int:
        n = C.c_int64(0)
        check(lib.obgpu_cg_bitmap_popcnt(self._h, lo, self.n_rows if hi is None else hi, C.byref(n)), "obgpu_cg_bitmap_popcnt", self.ctx._h)
        return n.value

    def fetch(self, lo: int = 0, count: Optional[int] = None) -> np.ndarray:
        count = self.n_rows - lo if count is None else count
        out = np.zeros(max(count, 1), dtype=np.uint8)
        check(lib.obgpu_cg_bitmap_fetch(self._h, lo, count, out.ctypes.data), "obgpu_cg_bitmap_fetch", self.ctx._h)
        return out[:count]

    def free(self):
        if self._h and self.ctx._h:
            lib.obgpu_cg_bitmap_free(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class ScanResult:
    """obgpu_result: device-resident dense output of one fused scan."""

    def __init__(self, batch: PageBatch, handle, n_proj):
        self.batch = batch
        self._h = handle
        self.n_proj = n_proj
        self._info = None

    def info(self) -> capi.ResultInfo:
        """Synchronises and returns totals; raises ObGpuError (e.g. OB_BUF_NOT_ENOUGH, OB_NOT_SUPPORTED)."""
        if self._info is None:
            info = capi.ResultInfo()
            code = lib.obgpu_result_info_get(self._h, C.byref(info))
            self._info = info
            check(code, "obgpu_scan (device status)", self.batch.ctx._h)
        return self._info

    @property
    def selected_rows(self) -> int:
        return self.info().selected_rows

    def col(self, i) -> capi.ResultCol:
        c = capi.ResultCol()
        check(lib.obgpu_result_col_get(self._h, i, C.byref(c)), "obgpu_result_col_get", self.batch.ctx._h)
        return c

    def fetch_col(self, i, row_begin=0, row_count=None, out=None, out_aux=None, out_nulls=None):
        """Device->host copy of column i. Returns (data, aux(lens) or None, nulls words)."""
        c = self.col(i)
        if row_count is None:
            row_count = self.selected_rows - row_begin
        dt = {8: np.uint64, 4: np.uint32, 1: np.uint8}[c.elem_len]
        data = np.zeros(max(row_count, 1), dtype=dt) if out is None else out
        aux = (np.zeros(max(row_count, 1), dtype=np.int32) if out_aux is None else out_aux) if c.is_string else None
        nulls = np.zeros(max((row_count + 63) // 64, 1), dtype=np.uint64) if out_nulls is None else out_nulls
        check(lib.obgpu_result_fetch_col(self._h, i, row_begin, row_count, data.ctypes.data,
                                         aux.ctypes.data if aux is not None else None, nulls.ctypes.data),
              "obgpu_result_fetch_col", self.batch.ctx._h)
        return data[:row_count], (aux[:row_count] if aux is not None else None), nulls[:(row_count + 63) // 64]

    def fetch_strings(self, i, row_begin=0, row_count=None):
        """obgpu_result_fetch_strings: (heap uint8, offsets int64 [n + 1]) -- the bytes of projected string column i."""
        if row_count is None:
            row_count = self.selected_rows - row_begin
        off = np.zeros(row_count + 1, dtype=np.int64)
        need = C.c_int64(0)
        heap = np.zeros(1, dtype=np.uint8)
        rc = lib.obgpu_result_fetch_strings(self._h, i, row_begin, row_count, heap.ctypes.data, 0, off.ctypes.data, C.byref(need))
        if rc == capi.OB_BUF_NOT_ENOUGH:
            heap = np.zeros(max(need.value, 1), dtype=np.uint8)
            rc = lib.obgpu_result_fetch_strings(self._h, i, row_begin, row_count, heap.ctypes.data, heap.size, off.ctypes.data, C.byref(need))
        check(rc, "obgpu_result_fetch_strings", self.batch.ctx._h)
        return heap[:need.value], off

    def group_by(self, group_col, aggs):
        """GROUP BY over every block of the scan, the rows the filter selected (one launch): returns (group_off int64
        [n_blocks + 1], out int64 [n_aggs][total groups][2]); block b's groups are its dictionary entries + the NULL group."""
        nb = self.batch.n_blocks
        goff = np.zeros(nb + 1, dtype=np.int64)
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        total = C.c_int64(0)
        dummy = np.zeros((len(aggs), 1, 2), dtype=np.int64)
        rc = lib.obgpu_result_group_by(self._h, group_col, spec.ctypes.data, len(aggs), goff.ctypes.data, dummy.ctypes.data, 0, C.byref(total))
        if rc != capi.OB_BUF_NOT_ENOUGH:
            check(rc, "obgpu_result_group_by", self.batch.ctx._h)
        out = np.zeros((len(aggs), max(total.value, 1), 2), dtype=np.int64)
        check(lib.obgpu_result_group_by(self._h, group_col, spec.ctypes.data, len(aggs), goff.ctypes.data, out.ctypes.data,
                                        max(total.value, 1), C.byref(total)), "obgpu_result_group_by", self.batch.ctx._h)
        return goff, out[:, :total.value]

    def group_by_values(self, group_col, aggs):
        """GROUP BY over every block of the scan with one group per distinct value of group_col (obgpu_result_group_by_values):
        returns (keys, out). keys: one per group in ascending order -- Python ints in the column's value domain (unsigned
        types non-negative) or bytes -- and None for the NULL group, which comes last; out: int64 [n_aggs][n_groups][2]."""
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        ng, kb, hn = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        check(lib.obgpu_result_group_by_values(self._h, group_col, spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb), C.byref(hn)),
              "obgpu_result_group_by_values", self.batch.ctx._h)
        n = ng.value
        keys = np.zeros(n + 1, dtype=np.int64)
        heap = np.zeros(max(kb.value, 1), dtype=np.uint8)
        out = np.zeros((len(aggs), max(n, 1), 2), dtype=np.int64)
        check(lib.obgpu_result_fetch_groups(self._h, keys.ctypes.data, heap.ctypes.data, out.ctypes.data), "obgpu_result_fetch_groups",
              self.batch.ctx._h)
        obj_type, dlen = C.c_int32(0), C.c_int32(0)
        check(lib.obgpu_batch_column_type(self.batch._h, group_col, C.byref(obj_type), C.byref(dlen)), "obgpu_batch_column_type",
              self.batch.ctx._h)
        if dlen.value == 0:
            vals = [bytes(heap[keys[g]:keys[g + 1]]) for g in range(n)]
        else:
            vals = [int(v) for v in keys[:n].tolist()]
            if obj_type.value in (capi.OBJ_UINT64, capi.OBJ_UINT32, capi.OBJ_UTINYINT, capi.OBJ_USMALLINT, capi.OBJ_UMEDIUMINT, capi.OBJ_YEAR):
                vals = [v & ((1 << 64) - 1) for v in vals]
        if hn.value:
            vals[-1] = None
        return vals, out[:, :n]

    def group_by_columns(self, group_cols, aggs):
        """GROUP BY over every block of the scan with one group per distinct tuple of values of group_cols (1..4 columns,
        obgpu_result_group_by_columns): returns (keys, out). keys: one tuple per group, in lexicographic order over group_cols,
        each element a Python int in its column's value domain (unsigned types non-negative), bytes, or None for NULL (last
        within its column); out: int64 [n_aggs][n_groups][2]."""
        cols = np.array(list(group_cols), dtype=np.int32)
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        ng, kb = C.c_int64(0), C.c_int64(0)
        check(lib.obgpu_result_group_by_columns(self._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb)),
              "obgpu_result_group_by_columns", self.batch.ctx._h)
        return self._fetch_group_columns(cols, len(aggs), ng.value, kb.value)

    def group_by_any(self, group_cols, aggs):
        """GROUP BY group_cols of any encoding (obgpu_result_group_by_any): returns (keys, out, path), keys and out as
        group_by_columns returns them (and byte for byte its groups wherever it accepts the batch), path capi.GROUP_PATH_DICT
        or capi.GROUP_PATH_CELLS: the fold the library chose."""
        cols = np.array(list(group_cols), dtype=np.int32)
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        ng, kb, path = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        check(lib.obgpu_result_group_by_any(self._h, cols.ctypes.data, len(cols), spec.ctypes.data, len(aggs), C.byref(ng), C.byref(kb),
                                            C.byref(path)), "obgpu_result_group_by_any", self.batch.ctx._h)
        keys, out = self._fetch_group_columns(cols, len(aggs), ng.value, kb.value)
        return keys, out, path.value

    def _fetch_group_columns(self, cols, n_aggs, n, key_bytes):
        nc = len(cols)
        keys = np.zeros((nc, n + 1), dtype=np.int64)
        nulls = np.zeros((nc, max(n, 1)), dtype=np.uint8)
        heap = np.zeros(max(key_bytes, 1), dtype=np.uint8)
        out = np.zeros((n_aggs, max(n, 1), 2), dtype=np.int64)
        check(lib.obgpu_result_fetch_group_columns(self._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data),
              "obgpu_result_fetch_group_columns", self.batch.ctx._h)
        types = []
        for gc in cols.tolist():
            obj_type, dlen = C.c_int32(0), C.c_int32(0)
            check(lib.obgpu_batch_column_type(self.batch._h, gc, C.byref(obj_type), C.byref(dlen)), "obgpu_batch_column_type",
                  self.batch.ctx._h)
            types.append((obj_type.value, dlen.value))
        return group_tuples(keys, nulls, heap, n, types), out[:, :n]

    def top_rows(self, keys, out_cols, k):
        """ORDER BY keys LIMIT k over every block of the scan (obgpu_result_top_rows): the first min(k, selected) selected rows.
        keys: 1..4 sort keys, each a store column or a (col, desc, nulls_first) tuple (ascending, NULLs last by default);
        out_cols: 0..16 store columns. Returns (positions, rows): positions one (block, block-relative row) per row, in order;
        rows one tuple per row, the out_cols values as Python ints in their column's value domain (unsigned types
        non-negative), bytes, or None for NULL. Ties are ordered by position."""
        karr, cols = sort_keys(keys), np.array(list(out_cols), dtype=np.int32)
        nr, hb = C.c_int64(0), C.c_int64(0)
        check(lib.obgpu_result_top_rows(self._h, karr.ctypes.data, len(karr), cols.ctypes.data if len(cols) else None, len(cols), k,
                                        C.byref(nr), C.byref(hb)), "obgpu_result_top_rows", self.batch.ctx._h)
        types = []
        for oc in cols.tolist():
            obj_type, dlen = C.c_int32(0), C.c_int32(0)
            check(lib.obgpu_batch_column_type(self.batch._h, oc, C.byref(obj_type), C.byref(dlen)), "obgpu_batch_column_type",
                  self.batch.ctx._h)
            types.append((obj_type.value, dlen.value))
        return fetch_top_rows(lambda *a: check(lib.obgpu_result_fetch_top_rows(self._h, *a), "obgpu_result_fetch_top_rows",
                                               self.batch.ctx._h), nr.value, hb.value, types)

    def fetch_datums(self, i, row_begin=0, row_count=None):
        """Column i as ObDatum[] (datum format): (datums structured array, slots uint64 array or None for strings)."""
        c = self.col(i)
        if row_count is None:
            row_count = self.selected_rows - row_begin
        datums = np.zeros(max(row_count, 1), dtype=DATUM_DTYPE)
        slots = None if c.is_string else np.zeros(max(row_count, 1), dtype=np.uint64)
        check(lib.obgpu_result_fetch_datums(self._h, i, row_begin, row_count, datums.ctypes.data,
                                            slots.ctypes.data if slots is not None else None), "obgpu_result_fetch_datums",
              self.batch.ctx._h)
        return datums[:row_count], (slots[:row_count] if slots is not None else None)

    def fetch_cols(self, idxs, row_begin=0, row_count=None, outs=None, out_nulls=None):
        """Several integer-class columns with one synchronisation (obgpu_result_fetch_cols). Returns
        ([data], [nulls words]); outs / out_nulls: optional preallocated (pinned) arrays per column."""
        if row_count is None:
            row_count = self.selected_rows - row_begin
        n = len(idxs)
        cols = [self.col(i) for i in idxs]
        datas, nulls = [], []
        for k, c in enumerate(cols):
            if c.is_string:
                raise ValueError("fetch_cols handles integer-class columns; use fetch_col for strings")
            dt = {8: np.uint64, 4: np.uint32, 1: np.uint8}[c.elem_len]
            datas.append(np.empty(max(row_count, 1), dtype=dt) if outs is None else outs[k])
            nulls.append(np.zeros(max((row_count + 63) // 64, 1), dtype=np.uint64) if out_nulls is None else out_nulls[k])
        ci = (C.c_int32 * max(n, 1))(*idxs)
        hd = (C.c_void_p * max(n, 1))(*[d.ctypes.data for d in datas])
        hn = (C.c_void_p * max(n, 1))(*[x.ctypes.data for x in nulls])
        check(lib.obgpu_result_fetch_cols(self._h, n, ci, row_begin, row_count, hd, None, hn), "obgpu_result_fetch_cols",
              self.batch.ctx._h)
        return [d[:row_count] for d in datas], [x[:(row_count + 63) // 64] for x in nulls]

    def skip_info(self):
        """(always-false blocks, always-true blocks) the skip index decided in this scan."""
        f, t = C.c_int64(0), C.c_int64(0)
        check(lib.obgpu_result_skip_info(self._h, C.byref(f), C.byref(t)), "obgpu_result_skip_info", self.batch.ctx._h)
        return f.value, t.value

    def aggregate(self, kind: int, col_a: int, col_b: int = -1):
        """Pushed-down aggregate over the selected rows (obgpu_result_aggregate). SUM / SUM_PRODUCT return a
        Python int (128-bit exact), COUNT an int, MIN / MAX an int or None when every row is NULL."""
        out = (C.c_int64 * 2)()
        check(lib.obgpu_result_aggregate(self._h, kind, col_a, col_b, out), "obgpu_result_aggregate", self.batch.ctx._h)
        lo, hi = int(out[0]), int(out[1])
        if kind in (capi.AGG_SUM, capi.AGG_SUM_PRODUCT):
            return (hi << 64) | (lo & ((1 << 64) - 1))
        if kind in (capi.AGG_MIN, capi.AGG_MAX):
            if not hi:
                return None
            return lo if self.col(col_a).obj_type not in (capi.OBJ_UINT64, capi.OBJ_UINT32, capi.OBJ_UTINYINT,
                                                          capi.OBJ_USMALLINT, capi.OBJ_UMEDIUMINT) else lo & ((1 << 64) - 1)
        return lo

    def fetch_sel_offsets(self) -> np.ndarray:
        out = np.zeros(self.batch.n_blocks + 1, dtype=np.int64)
        check(lib.obgpu_result_fetch_sel_offsets(self._h, out.ctypes.data), "obgpu_result_fetch_sel_offsets",
              self.batch.ctx._h)
        return out

    def fetch_row_ids(self, row_begin=0, row_count=None) -> np.ndarray:
        if row_count is None:
            row_count = self.selected_rows - row_begin
        out = np.zeros(max(row_count, 1), dtype=np.int32)
        check(lib.obgpu_result_fetch_row_ids(self._h, row_begin, row_count, out.ctypes.data),
              "obgpu_result_fetch_row_ids", self.batch.ctx._h)
        return out[:row_count]

    def fetch_bitmap(self, block, start=0, count=None) -> np.ndarray:
        if count is None:
            count = self.batch.block_info(block)[0] - start
        out = np.zeros(max(count, 1), dtype=np.uint8)
        check(lib.obgpu_result_fetch_bitmap(self._h, block, start, count, out.ctypes.data),
              "obgpu_result_fetch_bitmap", self.batch.ctx._h)
        return out[:count]

    def free(self):
        if self._h:
            if self.batch.ctx._h:
                lib.obgpu_result_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class GroupAccumulator:
    """obgpu_groups: the groups of several scan results (any page batches, any ctx of the device) merged by value on the device.
    fetch() returns (keys, out) in exactly ScanResult.group_by_columns' shape: what that call returns over all the added rows
    as one batch."""

    def __init__(self, handle, n_group_cols: int, n_aggs: int, owner, ctx: Optional[ScanContext] = None):
        self._h = handle
        self.n_cols, self.n_aggs = n_group_cols, n_aggs
        self.owner = owner   # what its ctx belongs to (a ScanContext or a HostScanPipeline): freed only while that is open
        self.ctx = ctx

    @classmethod
    def create(cls, ctx: ScanContext, n_group_cols: int, aggs):
        spec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        h = C.c_void_p()
        check(lib.obgpu_groups_create(ctx._h, n_group_cols, spec.ctypes.data if len(aggs) else None, len(aggs), C.byref(h)),
              "obgpu_groups_create", ctx._h)
        return cls(h, n_group_cols, len(aggs), ctx, ctx)

    def add(self, result: "ScanResult"):
        """Merge the result's current groups in; the result may be freed afterwards."""
        check(lib.obgpu_groups_add(self._h, result._h), "obgpu_groups_add", result.batch.ctx._h)

    def info(self):
        """(n_groups, key_bytes, [(obj_type, datum_len) per group column])"""
        ng, kb = C.c_int64(0), C.c_int64(0)
        types, lens = np.zeros(4, dtype=np.int32), np.zeros(4, dtype=np.int32)
        check(lib.obgpu_groups_info(self._h, C.byref(ng), C.byref(kb), types.ctypes.data, lens.ctypes.data), "obgpu_groups_info",
              self.ctx._h if self.ctx else None)
        return ng.value, kb.value, list(zip(types[:self.n_cols].tolist(), lens[:self.n_cols].tolist()))

    def fetch_raw(self):
        """(keys int64 [n_cols][n + 1], nulls uint8 [n_cols][n], heap uint8, out int64 [n_aggs][n][2]): the host layout of
        obgpu_result_fetch_group_columns."""
        n, kb, _ = self.info()
        keys = np.zeros((self.n_cols, n + 1), dtype=np.int64)
        nulls = np.zeros((self.n_cols, max(n, 1)), dtype=np.uint8)
        heap = np.zeros(max(kb, 1), dtype=np.uint8)
        out = np.zeros((self.n_aggs, max(n, 1), 2), dtype=np.int64)
        check(lib.obgpu_groups_fetch(self._h, keys.ctypes.data, nulls.ctypes.data, heap.ctypes.data, out.ctypes.data), "obgpu_groups_fetch",
              self.ctx._h if self.ctx else None)
        return keys, nulls[:, :n], heap[:kb], out[:, :n]

    def fetch(self):
        n, _, types = self.info()
        keys, nulls, heap, out = self.fetch_raw()
        return group_tuples(keys, nulls, heap, n, types), out

    def free(self):
        if self._h:
            if self.owner._h:
                lib.obgpu_groups_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
