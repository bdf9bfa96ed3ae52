"""Host-buffer scan pipeline: micro-blocks in host memory in, vectors in host memory out.

Thin binding of include/obgpu_pipeline.h (oceanbase_b200/csrc/host_pipeline.h): the host image is cut into page batches
of consecutive micro-blocks; n_streams worker threads of the LIBRARY, each with its own obgpu_ctx (= its own CUDA
stream), run open (H2D + index) -> scan -> fetch (D2H) of different batches concurrently, so the copies overlap in both
PCIe directions while the kernels slot in between. Results are delivered per batch in block order (dense inside a
batch), which is how a block-at-a-time consumer such as ObSSTableRowScanner drains them. Python only prepares the
spec and views the output buffers.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import capi
from .capi import lib
from .scan import GroupAccumulator, fetch_top_rows, flatten_filter, sort_keys
from .sstable import TableImage


@dataclass
class BatchOutput:
    block_begin: int
    block_end: int
    total_rows: int
    selected_rows: int
    cols: List[np.ndarray]           # per projected column: payload (uint64 / uint32 / uint8 views of the output buffers)
    lens: List[Optional[np.ndarray]]  # string columns: int32 lens
    nulls: List[np.ndarray]          # ObBitVector words of the batch's rows
    has_null: List[int]
    image_lo: int = 0                # byte offset of the batch's first block inside the caller's table image
    row_begin: int = 0               # first row of the batch inside the output buffers
    sources: list = field(default_factory=list)  # string columns: (array the pointers address, address of its byte 0), else None
    row_ids: Optional[np.ndarray] = None  # want_row_ids: int32 block-relative row id of every selected row of the batch

    def strings(self, c: int) -> List[Optional[bytes]]:
        """Cells of projected string column c as bytes (None for NULL rows), whether its pointers address the caller's image
        or a heap."""
        arr, base = self.sources[c]
        ptrs, lens, nulls = self.cols[c], self.lens[c], self.nulls[c]
        out = []
        for k in range(self.selected_rows):
            if (int(nulls[k >> 6]) >> (k & 63)) & 1:
                out.append(None)
                continue
            o = int(ptrs[k]) - base
            out.append(arr[o:o + int(lens[k])].tobytes())
        return out


def batch_bounds(n_blocks: int, blocks_per_batch: int, ramp: int = 0) -> List[int]:
    """Block index where every page batch starts (+ n_blocks at the end). ramp > 0: the first `ramp`
    batches are 1/2^ramp, ..., 1/2 of a full batch, so that the first results start flowing back (D2H)
    while most of the input is still on its way in. (Same cut as obpipe::batch_bounds.)"""
    bounds, b0 = [0], 0
    for k in range(ramp, 0, -1):
        step = max(1, blocks_per_batch >> k)
        if b0 + step >= n_blocks:
            break
        b0 += step
        bounds.append(b0)
    while b0 < n_blocks:
        b0 = min(n_blocks, b0 + blocks_per_batch)
        bounds.append(b0)
    return bounds


def split_table(table: TableImage, blocks_per_batch: int, ramp: int = 0) -> List[TableImage]:
    parts = []
    n = table.n_blocks
    bounds = batch_bounds(n, blocks_per_batch, ramp)
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        lo = int(table.offsets[b0])
        hi = int(table.offsets[b1]) if b1 < n else int(table.image.size)
        part = TableImage(table.image[lo:hi], table.offsets[b0:b1] - lo, table.sizes[b0:b1], 0, table.n_cols)
        part.image_lo = lo   # byte offset of the part inside the caller's table image (string pointers are rebased by it)
        parts.append(part)
    return parts


@dataclass
class HostOutputs:
    """Caller-owned output buffers of one pipelined scan (numpy views; allocate them pinned for speed)."""
    cap_rows: int
    data: List[np.ndarray]                 # per column: uint8 bytes, cap_rows * elem_bytes
    lens: List[Optional[np.ndarray]]       # int32[cap_rows] for string columns
    nulls: List[np.ndarray]                # uint64[cap_rows / 64]
    elem_bytes: List[int]
    keep: list = field(default_factory=list)
    heaps: List[Optional[np.ndarray]] = field(default_factory=list)  # string columns in heap mode: uint8 bytes of their cells

    @staticmethod
    def allocate(cap_rows: int, is_string: Sequence[bool], elem_len: Sequence[int], pinned: bool = False,
                 heap_bytes: Optional[int] = None) -> "HostOutputs":
        """heap_bytes: every string column gets a heap of that many bytes (its pointers then address the heap); None: none."""
        cap_rows = (int(cap_rows) + 63) // 64 * 64
        keep = []

        def buf(nbytes):
            if pinned:
                import torch
                t = torch.zeros(max(nbytes, 64), dtype=torch.uint8, pin_memory=True)
                keep.append(t)
                return t.numpy()
            return np.zeros(max(nbytes, 64), dtype=np.uint8)
        eb = [8 if s else int(l) for s, l in zip(is_string, elem_len)]
        data = [buf(cap_rows * e) for e in eb]
        lens = [buf(cap_rows * 4).view(np.int32) if s else None for s in is_string]
        nulls = [buf(cap_rows // 8).view(np.uint64) for _ in eb]
        heaps = [buf(int(heap_bytes)) if (s and heap_bytes is not None) else None for s in is_string]
        return HostOutputs(cap_rows, data, lens, nulls, eb, keep, heaps)


@dataclass
class HostScanOutput:
    batches: List[BatchOutput]
    total_rows: int
    selected_rows: int
    aggregates: list
    h2d_bytes: int
    d2h_bytes: int
    kernel_launches: int
    block_begin: Optional[np.ndarray] = None  # want_block_tables: int64 [n_blocks] output row where block i's selected rows start
    block_count: Optional[np.ndarray] = None  # ... and int64 [n_blocks] how many there are


@dataclass
class GroupByStats:
    """What obgpu_pipeline_group_by reports besides the groups: the batch cut and totals, as obgpu_pipeline_scan reports them."""
    n_batches: int
    batch_block_begin: np.ndarray    # int32 [n_batches + 1]
    batch_rows: np.ndarray           # int64 [n_batches]: selected rows of every batch
    total_rows: int
    selected_rows: int
    h2d_bytes: int
    d2h_bytes: int
    kernel_launches: int


def plan(table: TableImage, blocks_per_batch: int, selectivity_hint: float, ramp: int = 0):
    """obgpu_pipeline_plan: (number of page batches, rows the output buffers need for the planned slices). Reads only the
    blocks' headers in host memory: no device is needed."""
    spec, keep = HostScanPipeline._spec(table, None, [], blocks_per_batch, selectivity_hint, ramp, 0, None, None)
    nb, cap = C.c_int32(0), C.c_int64(0)
    capi.check(lib.obgpu_pipeline_plan(C.byref(spec), C.byref(nb), C.byref(cap)), "obgpu_pipeline_plan")
    return nb.value, cap.value


class _HeapOverflow(Exception):
    def __init__(self, used):
        self.used = used


class HostScanPipeline:
    """obgpu_pipeline: n_streams contexts (streams) created once, reused by every scan."""

    def __init__(self, device: int, n_workers: int = 3):
        self.device = device
        self._h = C.c_void_p()
        code = lib.obgpu_pipeline_create(device, n_workers, C.byref(self._h))
        if code != capi.OB_SUCCESS:
            raise capi.ObGpuError(code, "obgpu_pipeline_create", "no usable CUDA device; there is no CPU fallback")
        self.n_workers = n_workers
        self.launch_count = 0

    def close(self):
        if self._h:
            lib.obgpu_pipeline_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _spec(table, filter, proj, blocks_per_batch, selectivity_hint, ramp, string_base, agg_rows, agg_off):
        spec = capi.HostScanSpec()
        keep = []
        offs = np.ascontiguousarray(table.offsets, dtype=np.int64)
        sizes = np.ascontiguousarray(table.sizes, dtype=np.int64)
        keep += [offs, sizes]
        spec.image, spec.image_size = table.image.ctypes.data, table.image.size
        spec.offsets, spec.sizes, spec.n_blocks = offs.ctypes.data, sizes.ctypes.data, len(offs)
        f, fkeep = flatten_filter(filter)
        keep.append((f, fkeep))
        spec.filter = C.pointer(f) if f is not None else None
        pc = (C.c_int32 * max(len(proj), 1))(*proj)
        keep.append(pc)
        spec.proj_cols, spec.n_proj = pc, len(proj)
        spec.blocks_per_batch, spec.ramp = int(blocks_per_batch), int(ramp)
        spec.selectivity_hint, spec.string_base = float(selectivity_hint), int(string_base)
        if agg_rows is not None:
            ar = np.ascontiguousarray(agg_rows, dtype=np.uint8)
            ao = np.ascontiguousarray(agg_off, dtype=np.int64)
            assert len(ao) == table.n_blocks + 1
            keep += [ar, ao]
            spec.agg_rows, spec.agg_off = ar.ctypes.data, ao.ctypes.data
        return spec, keep

    def plan(self, table, filter, proj, blocks_per_batch, selectivity_hint, ramp=0):
        """(number of page batches, rows the output buffers need for the planned slices)."""
        return plan(table, blocks_per_batch, selectivity_hint, ramp)

    def scan(self, table: TableImage, filter, proj: Sequence[int], blocks_per_batch: int, selectivity_hint: float,
             outputs: Optional[HostOutputs] = None, string_base: int = 0, ramp: int = 0,
             agg_rows: Optional[np.ndarray] = None, agg_off: Optional[np.ndarray] = None,
             aggs: Sequence[tuple] = (), no_row_output: bool = False, proj_is_string: Optional[Sequence[bool]] = None,
             proj_elem_len: Optional[Sequence[int]] = None, zero_copy: bool = False, compressor: int = 0,
             heap_bytes: Optional[int] = None, want_row_ids: bool = False, want_block_tables: bool = False):
        """One pipelined scan of a host table. outputs=None: buffers are allocated here (pageable; spare room for every
        row, so slices that outgrow the selectivity hint always find a place). aggs: (kind, col_a, col_b) over the
        projected columns. Returns HostScanOutput; .batches views the output buffers.
        compressor (capi.COMPRESSOR_*): the blocks of `table` are in stored form (sstable.compress_table) and every page batch
        is decoded on the device; 0: plain blocks. heap_bytes: string cells come back as bytes in a heap per string column
        (BatchOutput.strings reads either mode); None: pointers into table.image, or, for stored blocks, heaps of 0 bytes.
        When outputs are allocated here, heap_bytes 0 sizes the heaps from the blocks' data_length_ sum and a heap that
        overflows is grown and the scan retried.
        want_row_ids: BatchOutput.row_ids holds the block-relative row id of every selected row (ObBitmap::get_row_ids).
        want_block_tables: HostScanOutput.block_begin / block_count say where each block's selected rows start in the output
        buffers and how many there are."""
        nproj = len(proj)
        if heap_bytes is None and compressor:
            heap_bytes = 0
        own = outputs is None and not no_row_output and nproj > 0
        heap_cap = None
        if own:
            if proj_is_string is None or proj_elem_len is None:
                proj_is_string, proj_elem_len = self._column_shapes(table, proj, compressor)
            if heap_bytes is not None:
                heap_cap = int(heap_bytes) or (int(sum(int(table.image[int(o) + 40:int(o) + 44].view(np.int32)[0]) for o in table.offsets)) + 64)
        for _ in range(16):
            try:
                return self._scan(table, filter, proj, blocks_per_batch, selectivity_hint, outputs, string_base, ramp, agg_rows, agg_off,
                                  aggs, no_row_output, proj_is_string, proj_elem_len, zero_copy, compressor, heap_cap, own,
                                  want_row_ids, want_block_tables)
            except _HeapOverflow as e:
                heap_cap = max(2 * heap_cap, 2 * e.used)
        raise capi.ObGpuError(capi.OB_BUF_NOT_ENOUGH, "obgpu_pipeline_scan", "string heaps kept overflowing")

    def _scan(self, table, filter, proj, blocks_per_batch, selectivity_hint, outputs, string_base, ramp, agg_rows, agg_off, aggs,
              no_row_output, proj_is_string, proj_elem_len, zero_copy, compressor, heap_cap, own, want_row_ids, want_block_tables):
        spec, keep = self._spec(table, filter, proj, blocks_per_batch, selectivity_hint, ramp, string_base, agg_rows, agg_off)
        nb, cap = C.c_int32(0), C.c_int64(0)
        capi.check(lib.obgpu_pipeline_plan(C.byref(spec), C.byref(nb), C.byref(cap)), "obgpu_pipeline_plan")
        nproj = len(proj)
        own_rows = 0
        if own or (want_row_ids and outputs is None):
            # spare room for every row, so slices that outgrow the selectivity hint always find a place
            total = int(sum(int(table.image[int(o) + 16:int(o) + 20].view(np.uint32)[0]) for o in table.offsets))
            own_rows = (cap.value + total + 64 * nb.value + 63) // 64 * 64
        if own:
            outputs = HostOutputs.allocate(own_rows, proj_is_string, proj_elem_len, heap_bytes=heap_cap)
        heap_used = np.zeros(max(nproj, 1), dtype=np.int64)
        heap_caps = None
        if outputs is not None and any(h is not None for h in outputs.heaps):
            oh = (C.c_void_p * max(nproj, 1))(*[(h.ctypes.data if h is not None else None) for h in outputs.heaps])
            heap_caps = np.array([(h.size if h is not None else 0) for h in outputs.heaps] or [0], dtype=np.int64)
            keep += [oh, heap_caps, heap_used]
            spec.out_heap, spec.out_heap_cap, spec.out_heap_used = oh, heap_caps.ctypes.data, heap_used.ctypes.data
        spec.compressor_type = int(compressor)
        if outputs is not None:
            od = (C.c_void_p * max(nproj, 1))(*[d.ctypes.data for d in outputs.data])
            ol = (C.c_void_p * max(nproj, 1))(*[(l.ctypes.data if l is not None else None) for l in outputs.lens])
            on = (C.c_void_p * max(nproj, 1))(*[x.ctypes.data for x in outputs.nulls])
            keep += [od, ol, on]
            spec.out_data, spec.out_lens, spec.out_nulls = od, ol, on
            spec.out_cap_rows = outputs.cap_rows
        row_ids = block_begin = block_count = None
        if want_row_ids:   # [out_cap_rows]: the row ids of batch b sit at its output rows
            if outputs is None:
                spec.out_cap_rows = own_rows
            row_ids = np.zeros(max(int(spec.out_cap_rows), 1), dtype=np.int32)
            spec.out_row_ids = row_ids.ctypes.data
        if want_block_tables:
            block_begin = np.zeros(table.n_blocks, dtype=np.int64)
            block_count = np.zeros(table.n_blocks, dtype=np.int64)
            spec.out_block_begin, spec.out_block_count = block_begin.ctypes.data, block_count.ctypes.data
        spec.no_row_output = 1 if no_row_output else 0
        spec.zero_copy = 1 if zero_copy else 0   # table.image must then be pinned host memory (the kernels read it over PCIe)
        if aggs:
            arr = (capi.HostAgg * len(aggs))()
            for i, (kind, a, b) in enumerate(aggs):
                arr[i].kind, arr[i].col_a, arr[i].col_b = kind, a, b
            keep.append(arr)
            spec.aggs, spec.n_aggs = arr, len(aggs)
        res = capi.HostScanResult()
        row_begin = np.zeros(nb.value + 1, dtype=np.int64)
        rows = np.zeros(nb.value + 1, dtype=np.int64)
        blk_begin = np.zeros(nb.value + 2, dtype=np.int32)
        res.batch_row_begin, res.batch_rows, res.batch_block_begin = row_begin.ctypes.data, rows.ctypes.data, blk_begin.ctypes.data
        res.n_batches_cap = nb.value
        code = lib.obgpu_pipeline_scan(self._h, C.byref(spec), C.byref(res))
        if code == capi.OB_BUF_NOT_ENOUGH and own and heap_caps is not None and (heap_used[:nproj] > heap_caps[:nproj]).any():
            raise _HeapOverflow(int(heap_used.max()))
        if code != capi.OB_SUCCESS:
            raise capi.ObGpuError(code, "obgpu_pipeline_scan", (lib.obgpu_pipeline_last_error(self._h) or b"").decode())
        self.launch_count += res.kernel_launches
        batches = []
        for b in range(res.n_batches):
            r0, n = int(row_begin[b]), int(rows[b])
            cols, lens, nulls, sources = [], [], [], []
            if outputs is not None and not no_row_output:
                for c in range(nproj):
                    heap = outputs.heaps[c] if outputs.heaps else None
                    if heap is not None:
                        sources.append((heap, heap.ctypes.data))
                    else:
                        sources.append((table.image, int(string_base)) if outputs.lens[c] is not None else None)
                    e = outputs.elem_bytes[c]
                    dt = {8: np.uint64, 4: np.uint32, 1: np.uint8}[e]
                    cols.append(outputs.data[c][r0 * e:(r0 + n) * e].view(dt))
                    lens.append(outputs.lens[c][r0:r0 + n] if outputs.lens[c] is not None else None)
                    nulls.append(outputs.nulls[c][r0 // 64:r0 // 64 + (n + 63) // 64])
            b0, b1 = int(blk_begin[b]), int(blk_begin[b + 1])
            batches.append(BatchOutput(b0, b1, 0, n, cols, lens, nulls, [int(x.any()) for x in nulls], int(table.offsets[b0]), r0,
                                       sources, row_ids[r0:r0 + n] if row_ids is not None else None))
        aggregates = []
        for i, (kind, a, b) in enumerate(aggs):
            lo, hi = int(res.agg_out[i][0]), int(res.agg_out[i][1])
            if kind in (capi.AGG_SUM, capi.AGG_SUM_PRODUCT):
                aggregates.append((hi << 64) | (lo & ((1 << 64) - 1)))
            elif kind in (capi.AGG_MIN, capi.AGG_MAX):
                aggregates.append(lo if hi else None)
            else:
                aggregates.append(lo)
        out = HostScanOutput(batches, int(res.total_rows), int(res.selected_rows), aggregates, int(res.h2d_bytes),
                             int(res.d2h_bytes), int(res.kernel_launches), block_begin, block_count)
        out._keep = (keep, outputs, row_ids)
        return out

    def group_by(self, table: TableImage, filter, group_cols: Sequence[int], aggs: Sequence[tuple], blocks_per_batch: int = 0,
                 ramp: int = 0, compressor: int = 0, zero_copy: bool = False, agg_rows: Optional[np.ndarray] = None,
                 agg_off: Optional[np.ndarray] = None):
        """GROUP BY group_cols (1..4 store indexes) over the rows of a host table that filter selects, every page batch grouped
        and its groups merged on the device (obgpu_pipeline_group_by). aggs: (kind, store col or -1) as
        ScanResult.group_by_columns takes them. Returns (keys, out, GroupByStats); keys and out are exactly what
        ScanResult.group_by_columns returns over the whole table as one batch. blocks_per_batch 0: n_blocks / 12."""
        keys, out, stats, _ = self._group_by("obgpu_pipeline_group_by", table, filter, group_cols, aggs, blocks_per_batch, ramp, compressor,
                                             zero_copy, agg_rows, agg_off)
        return keys, out, stats

    def group_by_any(self, table: TableImage, filter, group_cols: Sequence[int], aggs: Sequence[tuple], blocks_per_batch: int = 0,
                     ramp: int = 0, compressor: int = 0, zero_copy: bool = False, agg_rows: Optional[np.ndarray] = None,
                     agg_off: Optional[np.ndarray] = None):
        """group_by for group columns of any encoding (obgpu_pipeline_group_by_any): each batch grouped by
        ScanResult.group_by_any's path. Returns (keys, out, GroupByStats, cells_batches): keys and out are exactly what
        ScanResult.group_by_any returns over the whole table as one batch; cells_batches how many batches took the cells path."""
        return self._group_by("obgpu_pipeline_group_by_any", table, filter, group_cols, aggs, blocks_per_batch, ramp, compressor, zero_copy,
                              agg_rows, agg_off)

    def _group_by(self, entry, table, filter, group_cols, aggs, blocks_per_batch, ramp, compressor, zero_copy, agg_rows, agg_off):
        spec, keep = self._spec(table, filter, [], blocks_per_batch, 1.0, ramp, 0, agg_rows, agg_off)
        spec.no_row_output = 1
        spec.compressor_type = int(compressor)
        spec.zero_copy = 1 if zero_copy else 0   # table.image must then be pinned host memory (the kernels read it over PCIe)
        nb, cap = C.c_int32(0), C.c_int64(0)
        capi.check(lib.obgpu_pipeline_plan(C.byref(spec), C.byref(nb), C.byref(cap)), "obgpu_pipeline_plan")
        cols = np.array(list(group_cols), dtype=np.int32)
        gspec = np.array([(k, c) for k, c in aggs], dtype=np.int32).reshape(-1, 2)
        res = capi.HostScanResult()
        row_begin = np.zeros(nb.value + 1, dtype=np.int64)
        rows = np.zeros(nb.value + 1, dtype=np.int64)
        blk_begin = np.zeros(nb.value + 2, dtype=np.int32)
        res.batch_row_begin, res.batch_rows, res.batch_block_begin = row_begin.ctypes.data, rows.ctypes.data, blk_begin.ctypes.data
        res.n_batches_cap = nb.value
        h = C.c_void_p()
        args = [self._h, C.byref(spec), cols.ctypes.data, len(cols), gspec.ctypes.data if len(aggs) else None, len(aggs), C.byref(res),
                C.byref(h)]
        cells = C.c_int32(0)
        if entry == "obgpu_pipeline_group_by_any":
            args.append(C.byref(cells))
        code = getattr(lib, entry)(*args)
        if code != capi.OB_SUCCESS:
            raise capi.ObGpuError(code, entry, (lib.obgpu_pipeline_last_error(self._h) or b"").decode())
        self.launch_count += res.kernel_launches
        acc = GroupAccumulator(h, len(cols), len(aggs), self)
        try:
            keys, out = acc.fetch()
        finally:
            acc.free()
        n = res.n_batches
        stats = GroupByStats(n, blk_begin[:n + 1].copy(), rows[:n].copy(), int(res.total_rows), int(res.selected_rows), int(res.h2d_bytes),
                             int(res.d2h_bytes), int(res.kernel_launches))
        return keys, out, stats, cells.value

    def top_rows(self, table: TableImage, filter, keys, out_cols: Sequence[int], k: int, blocks_per_batch: int = 0, ramp: int = 0,
                 compressor: int = 0, zero_copy: bool = False, agg_rows: Optional[np.ndarray] = None, agg_off: Optional[np.ndarray] = None):
        """ORDER BY keys LIMIT k over the rows of a host table that filter selects, every page batch's rows merged on the device
        (obgpu_pipeline_top_rows). keys and out_cols as ScanResult.top_rows takes them. Returns (positions, rows, stats):
        positions one (block index in the table, row) per row; positions and rows are exactly what ScanResult.top_rows returns
        over the whole table as one batch. blocks_per_batch 0: n_blocks / 12."""
        spec, keep = self._spec(table, filter, [], blocks_per_batch, 1.0, ramp, 0, agg_rows, agg_off)
        spec.no_row_output = 1
        spec.compressor_type = int(compressor)
        spec.zero_copy = 1 if zero_copy else 0
        nb, cap = C.c_int32(0), C.c_int64(0)
        capi.check(lib.obgpu_pipeline_plan(C.byref(spec), C.byref(nb), C.byref(cap)), "obgpu_pipeline_plan")
        karr, cols = sort_keys(keys), np.array(list(out_cols), dtype=np.int32)
        res = capi.HostScanResult()
        row_begin = np.zeros(nb.value + 1, dtype=np.int64)
        rows = np.zeros(nb.value + 1, dtype=np.int64)
        blk_begin = np.zeros(nb.value + 2, dtype=np.int32)
        res.batch_row_begin, res.batch_rows, res.batch_block_begin = row_begin.ctypes.data, rows.ctypes.data, blk_begin.ctypes.data
        res.n_batches_cap = nb.value
        nr, hb = C.c_int64(0), C.c_int64(0)
        code = lib.obgpu_pipeline_top_rows(self._h, C.byref(spec), karr.ctypes.data, len(karr), cols.ctypes.data if len(cols) else None,
                                           len(cols), k, C.byref(res), C.byref(nr), C.byref(hb))
        if code != capi.OB_SUCCESS:
            raise capi.ObGpuError(code, "obgpu_pipeline_top_rows", (lib.obgpu_pipeline_last_error(self._h) or b"").decode())
        self.launch_count += res.kernel_launches

        def fetch(*a):
            capi.check(lib.obgpu_pipeline_fetch_top_rows(self._h, *a), "obgpu_pipeline_fetch_top_rows")
        positions, out = fetch_top_rows(fetch, nr.value, hb.value, self._column_types(table, cols.tolist(), compressor))
        n = res.n_batches
        stats = GroupByStats(n, blk_begin[:n + 1].copy(), rows[:n].copy(), int(res.total_rows), int(res.selected_rows), int(res.h2d_bytes),
                             int(res.d2h_bytes), int(res.kernel_launches))
        return positions, out, stats

    def _column_types(self, table, cols, compressor=0):
        """(obj_type, datum length; 0 for strings) of columns, read from the first block's column headers, or from the block
        opened on the device when it is stored compressed"""
        from .capi import OBJ_VARCHAR, OBJ_CHAR
        if compressor:
            from .scan import PageBatch, ScanContext
            from .sstable import TableImage as _T
            ctx = ScanContext(self.device)
            o, n = int(table.offsets[0]), int(table.sizes[0])
            one = _T(np.ascontiguousarray(table.image[o:o + n]), np.zeros(1, dtype=np.int64), np.array([n], dtype=np.int64), 0, table.n_cols)
            batch = PageBatch(ctx, one, compressor=compressor)
            out = []
            try:
                for c in cols:
                    t, dl = C.c_int32(0), C.c_int32(0)
                    capi.check(lib.obgpu_batch_column_type(batch._h, c, C.byref(t), C.byref(dl)), "obgpu_batch_column_type", ctx._h)
                    out.append((t.value, dl.value))
            finally:
                batch.close()
                ctx.close()
            return out
        blk = table.block(0)
        hs = int(blk[4:8].view(np.uint32)[0])
        cs = int(blk[20]) == 3
        out = []
        for c in cols:
            t = int(blk[hs + 12 + 4 * c + 3]) if cs else int(blk[hs + 16 * c + 3])
            out.append((t, 0 if t in (OBJ_VARCHAR, OBJ_CHAR) else capi.datum_len_of(t)))
        return out

    def _column_shapes(self, table, proj, compressor=0):
        """(is_string, elem_len) of the projected columns, read from the first block's column headers. A stored block's
        headers may be compressed: the block is then opened on the device and asked."""
        from .capi import OBJ_VARCHAR, OBJ_CHAR
        if compressor:
            from .scan import PageBatch, ScanContext
            from .sstable import TableImage as _T
            ctx = ScanContext(self.device)
            o, n = int(table.offsets[0]), int(table.sizes[0])
            one = _T(np.ascontiguousarray(table.image[o:o + n]), np.zeros(1, dtype=np.int64), np.array([n], dtype=np.int64), 0, table.n_cols)
            batch = PageBatch(ctx, one, compressor=compressor)
            is_str, elem = [], []
            try:
                for c in proj:
                    t, dl = C.c_int32(0), C.c_int32(0)
                    capi.check(lib.obgpu_batch_column_type(batch._h, c, C.byref(t), C.byref(dl)), "obgpu_batch_column_type", ctx._h)
                    is_str.append(dl.value == 0)
                    elem.append(8 if dl.value == 0 else dl.value)
            finally:
                batch.close()
                ctx.close()
            return is_str, elem
        blk = table.block(0)
        hs = int(blk[4:8].view(np.uint32)[0])
        cs = int(blk[20]) == 3
        is_str, elem = [], []
        for c in proj:
            t = int(blk[hs + 12 + 4 * c + 3]) if cs else int(blk[hs + 16 * c + 3])
            s = t in (OBJ_VARCHAR, OBJ_CHAR)
            is_str.append(s)
            elem.append(8 if s else capi.datum_len_of(t))
        return is_str, elem
