"""Synthetic SSTable construction on top of the host micro-block writer
(oceanbase_b200/csrc/sstable_writer.cpp; reference: ObMicroBlockEncoder::build_block,
encoding/ob_micro_block_encoder.cpp:561-721)."""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import capi
from .capi import lib, check


@dataclass
class Column:
    """One column of the table to encode.

    values: int64 ndarray for integer classes, or a sequence of bytes for string classes
    (alternatively pass str_heap / str_off directly for big string columns)."""
    obj_type: int
    encoding: int
    values: object = None
    nulls: Optional[np.ndarray] = None
    byte_packing_only: bool = False
    ref_col: int = 0   # ENC_COLUMN_EQUAL / ENC_COLUMN_SUBSTR: index of the referenced column
    str_heap: Optional[np.ndarray] = None
    str_off: Optional[np.ndarray] = None
    _keep: list = field(default_factory=list, repr=False)

    def is_string(self):
        return self.obj_type in (capi.OBJ_VARCHAR, capi.OBJ_CHAR)

    def to_input(self) -> capi.ColInput:
        ci = capi.ColInput()
        ci.obj_type = self.obj_type
        ci.encoding = self.encoding
        ci.byte_packing_only = 1 if self.byte_packing_only else 0
        ci.ref_col = int(self.ref_col)
        if self.is_string():
            if self.str_heap is None:
                vals = [b"" if v is None else bytes(v) for v in self.values]
                lens = np.fromiter((len(v) for v in vals), dtype=np.int64, count=len(vals))
                off = np.zeros(len(vals) + 1, dtype=np.int64)
                np.cumsum(lens, out=off[1:])
                heap = np.frombuffer(b"".join(vals) + b"\0", dtype=np.uint8).copy()
                self.str_heap, self.str_off = heap, off
            heap = np.ascontiguousarray(self.str_heap, dtype=np.uint8)
            off = np.ascontiguousarray(self.str_off, dtype=np.int64)
            self._keep += [heap, off]
            ci.str_heap = heap.ctypes.data
            ci.str_off = off.ctypes.data
        else:
            v = np.ascontiguousarray(self.values, dtype=np.int64)
            self._keep.append(v)
            ci.i64 = v.ctypes.data
        if self.nulls is not None:
            n = np.ascontiguousarray(self.nulls, dtype=np.uint8)
            self._keep.append(n)
            ci.is_null = n.ctypes.data
        return ci

    def nrows(self):
        if self.is_string():
            return (len(self.str_off) - 1) if self.str_off is not None else len(self.values)
        return len(self.values)


@dataclass
class TableImage:
    """Packed image of consecutive micro-blocks (the 'block cache' view the scan consumes)."""
    image: np.ndarray          # uint8
    offsets: np.ndarray        # int64 [n_blocks]
    sizes: np.ndarray          # int64 [n_blocks]
    total_rows: int
    n_cols: int
    image_lo: int = 0          # set by pipeline.split_table: offset of this part inside the table it was cut from

    @property
    def n_blocks(self):
        return len(self.offsets)

    def block(self, i) -> np.ndarray:
        return self.image[self.offsets[i]:self.offsets[i] + self.sizes[i]]

    @staticmethod
    def concat(parts: Sequence["TableImage"]) -> "TableImage":
        offs, pos = [], 0
        for p in parts:
            offs.append(p.offsets + pos)
            pos += len(p.image)
        return TableImage(np.concatenate([p.image for p in parts]), np.concatenate(offs),
                          np.concatenate([p.sizes for p in parts]), sum(p.total_rows for p in parts),
                          parts[0].n_cols)


def _inputs(cols: List[Column]):
    arr = (capi.ColInput * len(cols))()
    for i, c in enumerate(cols):
        arr[i] = c.to_input()
    return arr


def encode_block(cols: List[Column], row_begin=0, nrows=None, rowkey_cnt=0) -> np.ndarray:
    n = cols[0].nrows() - row_begin if nrows is None else nrows
    arr = _inputs(cols)
    size = C.c_int64(0)
    check(lib.obgpu_writer_encode_block(arr, len(cols), rowkey_cnt, row_begin, n, None, 0, C.byref(size)),
          "obgpu_writer_encode_block(size)")
    out = np.zeros(size.value, dtype=np.uint8)
    check(lib.obgpu_writer_encode_block(arr, len(cols), rowkey_cnt, row_begin, n, out.ctypes.data, out.size,
                                        C.byref(size)), "obgpu_writer_encode_block")
    return out


def encode_table(cols: List[Column], rows_per_block: int, rowkey_cnt=0, align=128, n_threads=0,
                 out: Optional[np.ndarray] = None) -> TableImage:
    total = cols[0].nrows()
    arr = _inputs(cols)
    h = C.c_void_p()
    check(lib.obgpu_writer_encode_table(arr, len(cols), rowkey_cnt, total, rows_per_block, align, n_threads,
                                        C.byref(h)), "obgpu_writer_encode_table")
    try:
        size, nb = C.c_int64(0), C.c_int32(0)
        check(lib.obgpu_table_image_info(h, C.byref(size), C.byref(nb)), "obgpu_table_image_info")
        image = np.empty(size.value, dtype=np.uint8) if out is None else out[:size.value]
        offsets = np.zeros(nb.value, dtype=np.int64)
        sizes = np.zeros(nb.value, dtype=np.int64)
        check(lib.obgpu_table_image_export(h, image.ctypes.data, image.size, offsets.ctypes.data,
                                           sizes.ctypes.data, nb.value), "obgpu_table_image_export")
    finally:
        lib.obgpu_table_image_free(h)
    return TableImage(image, offsets, sizes, total, len(cols))


# ---- macro blocks (ObMacroBlock, blocksstable/ob_macro_block.cpp) ---------------------------------------------------------------
@dataclass
class MacroImage:
    """Fixed-size macro blocks holding the micro-blocks of a TableImage back to back (no alignment inside a macro block)."""
    image: np.ndarray          # uint8, n_macro * macro_block_size
    macro_block_size: int
    n_macro: int
    first_micro: np.ndarray    # int32 [n_macro + 1]


def build_macro_blocks(table: TableImage, col_types: Sequence[int], rowkey_cnt: int, tablet_id: int = 200001, logical_version: int = 1,
                       first_data_seq: int = 0, header_version: int = 1, is_cg: bool = False, macro_block_size: int = 2 << 20,
                       col_orders: Optional[Sequence[int]] = None, compressor: Optional[int] = None) -> MacroImage:
    """ObMacroBlock::write_micro_block / write_macro_header over the micro-blocks of `table`.
    compressor (capi.COMPRESSOR_*): the plain blocks are compressed first (compress_table) and the macro headers record it."""
    if compressor is not None and compressor != capi.COMPRESSOR_NONE:
        table = compress_table(table, compressor)
    comp = capi.COMPRESSOR_NONE if compressor is None else int(compressor)
    n_cols = len(col_types)
    metas = np.zeros((n_cols, 4), dtype=np.uint8)
    metas[:, 0] = col_types
    orders = np.ascontiguousarray(col_orders if col_orders is not None else [0] * n_cols, dtype=np.int32)
    spec = capi.MacroSpec(tablet_id, logical_version, first_data_seq, header_version, 1 if is_cg else 0, rowkey_cnt, n_cols,
                          metas.ctypes.data, orders.ctypes.data, macro_block_size)
    img = np.ascontiguousarray(table.image)
    off = np.ascontiguousarray(table.offsets, dtype=np.int64)
    sz = np.ascontiguousarray(table.sizes, dtype=np.int64)
    # every macro block holds at least one micro-block: n_blocks macro blocks is the upper bound
    data_per_macro = macro_block_size - 24 - 128 - 16 * n_cols - 1
    est = int(sz.sum() // max(data_per_macro - int(sz.max()), 1)) + 2
    out = np.zeros(min(est, table.n_blocks) * macro_block_size, dtype=np.uint8)
    first = np.zeros(table.n_blocks + 1, dtype=np.int32)
    size, nm = C.c_int64(0), C.c_int32(0)
    check(lib.obgpu_writer_build_macro_blocks_ex(img.ctypes.data, off.ctypes.data, sz.ctypes.data, table.n_blocks, C.byref(spec),
                                                 out.ctypes.data, out.size, C.byref(size), C.byref(nm), first.ctypes.data, first.size,
                                                 comp), "obgpu_writer_build_macro_blocks_ex")
    return MacroImage(out[:size.value], macro_block_size, nm.value, first[:nm.value + 1].copy())


# ---- compressed micro-blocks (ObMicroBlockCompressor: plain header, payload compressed on its own) ----------------------------
def lz4_compress(data) -> np.ndarray:
    """One LZ4 block (block format, no frame) of `data` by the writer's compressor."""
    src = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data, dtype=np.uint8)
    n = C.c_int64(0)
    check(lib.obgpu_writer_lz4_compress(src.ctypes.data, src.size, None, 0, C.byref(n)), "obgpu_writer_lz4_compress(size)")
    out = np.zeros(max(n.value, 1), dtype=np.uint8)
    check(lib.obgpu_writer_lz4_compress(src.ctypes.data, src.size, out.ctypes.data, out.size, C.byref(n)), "obgpu_writer_lz4_compress")
    return out[:n.value]


def zstd_compress(data) -> np.ndarray:
    """One zstd frame (RFC 8878: Single_Segment, Frame_Content_Size, no checksum) of `data` by the writer's compressor."""
    src = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data, dtype=np.uint8)
    n = C.c_int64(0)
    check(lib.obgpu_writer_zstd_compress(src.ctypes.data, src.size, None, 0, C.byref(n)), "obgpu_writer_zstd_compress(size)")
    out = np.zeros(max(n.value, 1), dtype=np.uint8)
    check(lib.obgpu_writer_zstd_compress(src.ctypes.data, src.size, out.ctypes.data, out.size, C.byref(n)), "obgpu_writer_zstd_compress")
    return out[:n.value]


def zlib_compress(data) -> np.ndarray:
    """One zlib stream (RFC 1950: header 78 01, fixed-Huffman or stored blocks, Adler-32) of `data` by the writer's compressor."""
    src = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data, dtype=np.uint8)
    n = C.c_int64(0)
    check(lib.obgpu_writer_zlib_compress(src.ctypes.data, src.size, None, 0, C.byref(n)), "obgpu_writer_zlib_compress(size)")
    out = np.zeros(max(n.value, 1), dtype=np.uint8)
    check(lib.obgpu_writer_zlib_compress(src.ctypes.data, src.size, out.ctypes.data, out.size, C.byref(n)), "obgpu_writer_zlib_compress")
    return out[:n.value]


def compress_table(table: TableImage, compressor: int, align: int = 1) -> TableImage:
    """The blocks of `table` in stored form: each payload compressed with `compressor` (capi.COMPRESSOR_*) and kept raw when
    that is not smaller (data_zlength_, data_checksum_ and the header checksum follow). align=1: blocks back to back, at any
    byte offset, as inside a macro block."""
    img = np.ascontiguousarray(table.image)
    off = np.ascontiguousarray(table.offsets, dtype=np.int64)
    sz = np.ascontiguousarray(table.sizes, dtype=np.int64)
    cap = int(((sz + align - 1) // align * align).sum()) + align
    out = np.zeros(cap, dtype=np.uint8)
    o_off = np.zeros(table.n_blocks, dtype=np.int64)
    o_sz = np.zeros(table.n_blocks, dtype=np.int64)
    used = C.c_int64(0)
    check(lib.obgpu_writer_compress_blocks(img.ctypes.data, off.ctypes.data, sz.ctypes.data, table.n_blocks, int(compressor), align,
                                           out.ctypes.data, out.size, o_off.ctypes.data, o_sz.ctypes.data, C.byref(used)),
          "obgpu_writer_compress_blocks")
    return TableImage(out[:used.value], o_off, o_sz, table.total_rows, table.n_cols)


# ---- skip index: aggregate rows (include/obgpu_skip_index.h) -------------------------------------------------
def agg_row_write(cells, version: int = 3) -> np.ndarray:
    """ObAggRowWriter: cells = [(col_idx, col_type, value)] with value None (not stored), bytes, or
    (bytes, is_prefix)."""
    arr = (capi.AggCell * len(cells))()
    keep = []
    for i, (col_idx, col_type, value) in enumerate(cells):
        arr[i].col_idx, arr[i].col_type = col_idx, col_type
        if value is None:
            arr[i].is_null = 1
            continue
        data, prefix = value if isinstance(value, tuple) else (value, False)
        buf = C.create_string_buffer(bytes(data), max(len(data), 1))
        keep.append(buf)
        arr[i].data, arr[i].len, arr[i].is_prefix = C.addressof(buf), len(data), 1 if prefix else 0
    size = C.c_int64(0)
    check(lib.obgpu_agg_row_write(arr, len(cells), version, None, 0, C.byref(size)), "obgpu_agg_row_write(size)")
    out = np.zeros(size.value, dtype=np.uint8)
    check(lib.obgpu_agg_row_write(arr, len(cells), version, out.ctypes.data, out.size, C.byref(size)), "obgpu_agg_row_write")
    return out


def block_agg_row(cols: List[Column], agg_cols: Sequence[int], row_begin=0, nrows=None) -> np.ndarray:
    """MIN / MAX / NULL_COUNT of the listed columns over a row range, serialized (ObSkipIndexAggregator + ObAggRowWriter)."""
    n = cols[0].nrows() - row_begin if nrows is None else nrows
    arr = _inputs(cols)
    ac = np.ascontiguousarray(agg_cols, dtype=np.int32)
    size = C.c_int64(0)
    check(lib.obgpu_writer_block_agg_row(arr, len(cols), ac.ctypes.data, len(ac), row_begin, n, None, 0, C.byref(size)),
          "obgpu_writer_block_agg_row(size)")
    out = np.zeros(size.value, dtype=np.uint8)
    check(lib.obgpu_writer_block_agg_row(arr, len(cols), ac.ctypes.data, len(ac), row_begin, n, out.ctypes.data, out.size,
                                         C.byref(size)), "obgpu_writer_block_agg_row")
    return out


def table_agg_rows(cols: List[Column], agg_cols: Sequence[int], rows_per_block: int):
    """One aggregate row per block of encode_table's blocking: (bytes, offsets[n_blocks + 1])."""
    total = cols[0].nrows()
    arr = _inputs(cols)
    ac = np.ascontiguousarray(agg_cols, dtype=np.int32)
    nb = (total + rows_per_block - 1) // rows_per_block
    size = C.c_int64(0)
    check(lib.obgpu_writer_table_agg_rows(arr, len(cols), ac.ctypes.data, len(ac), total, rows_per_block, None, 0, None,
                                          C.byref(size)), "obgpu_writer_table_agg_rows(size)")
    out = np.zeros(max(size.value, 1), dtype=np.uint8)
    offs = np.zeros(nb + 1, dtype=np.int64)
    check(lib.obgpu_writer_table_agg_rows(arr, len(cols), ac.ctypes.data, len(ac), total, rows_per_block, out.ctypes.data,
                                          out.size, offs.ctypes.data, C.byref(size)), "obgpu_writer_table_agg_rows")
    return out[:size.value], offs
