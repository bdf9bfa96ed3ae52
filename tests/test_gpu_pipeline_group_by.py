"""GROUP BY through the host pipeline (obgpu_pipeline_group_by, HostScanPipeline.group_by) against the plain tuple model of the
generator's cells (test_gpu_group_by_columns.tuple_model): the groups of every page batch merged on the device are the groups of
the selected rows of the whole table.

Sweeps: batch sizes of 1, 3, 7, all and more than all blocks and the default; ramps 0 and 2; 1, 2 and 4 workers; no filter, a
selective filter and one that selects nothing; PAX and CS tables; LZ4-, zstd- and zlib-stored blocks; a zero-copy pinned image;
skip-index-pruned blocks; several workers folding at once in shared memory, each page batch with its own dictionary sizes
and so its own shared-memory size; a table whose dictionaries hold more than 65 536 values in all while every batch stays under
(test_pipeline_group_by_shapes proves the counts), next to one batch over; the refusals of a column that is not dictionary coded
and of row output; the result's totals and batch cut."""
import ctypes as C

import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM
from test_gpu_aggregate_exact import PATH_AGGS, PATH_ROWS, path_table
from test_gpu_group_by_columns import tuple_model
from test_gpu_group_by_values import path_cells
from test_pipeline_group_by_shapes import CAP_SPLIT, cap_split_cells, cap_split_table, vary_cells, vary_table
from test_scan_codes_model import auto_table, cs_table, string_table

pytestmark = pytest.mark.gpu

AGGS = [(COUNT, -1), (SUM, 1), (MIN, 3), (MAX, 3), (COUNT, 1)]
STR_AGGS = [(COUNT, -1), (SUM, 3), (MIN, 3), (MAX, 4), (COUNT, 4)]


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def pipes():
    from oceanbase_b200.pipeline import HostScanPipeline
    ps = {w: HostScanPipeline(0, n_workers=w) for w in (1, 2, 4)}
    yield ps
    for p in ps.values():
        p.close()


def assert_model(got, t, gcols, aggs, rows, what=""):
    keys, out, stats = got
    want_keys, want = tuple_model([t.cells[c] for c in gcols], list(rows), aggs, t.cells)
    assert keys == want_keys, what
    assert np.array_equal(out, want), what
    return stats


def assert_stats(stats, table, bpb, ramp, rows_sel, zero_copy=False):
    from oceanbase_b200.pipeline import batch_bounds
    n = table.n_blocks
    bounds = batch_bounds(n, bpb if bpb > 0 else max(1, n // 12), ramp)
    assert stats.n_batches == len(bounds) - 1
    assert stats.batch_block_begin.tolist() == bounds
    total = sum(int(table.image[int(o) + 16:int(o) + 20].view(np.uint32)[0]) for o in table.offsets)
    assert stats.total_rows == total and stats.selected_rows == len(rows_sel)
    sel = set(rows_sel)
    starts = [sum(int(table.image[int(o) + 16:int(o) + 20].view(np.uint32)[0]) for o in table.offsets[:b]) for b in bounds]
    assert stats.batch_rows.tolist() == [sum(1 for r in range(a, b) if r in sel) for a, b in zip(starts[:-1], starts[1:])]
    assert stats.h2d_bytes == (0 if zero_copy else table.image.size)
    assert stats.d2h_bytes == 0 and stats.kernel_launches > 0


# ---- batch cuts x ramps x workers x filters on a PAX and a CS table ------------------------------------------------------
@pytest.mark.parametrize("bpb", [1, 3, 7, "all", "more", 0])
@pytest.mark.parametrize("ramp", [0, 2])
def test_batch_cuts(ob, pipes, bpb, ramp):
    t = string_table()
    n = t.image.n_blocks
    b = {"all": n, "more": n + 5}.get(bpb, bpb)
    half = t.n // 2
    filters = [(None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half]),
               (ob.White(0, ob.WHITE_OP_LT, (0,)), [])]
    for i, (flt, rows) in enumerate(filters):
        for gcols in ([2, 1], [1, 2, 4]):
            p = pipes[(1, 2, 4)[(i + len(gcols)) % 3]]
            got = p.group_by(t.image, flt, gcols, STR_AGGS, blocks_per_batch=b, ramp=ramp)
            stats = assert_model(got, t, gcols, STR_AGGS, rows, (bpb, ramp, i, gcols))
            assert_stats(stats, t.image, b, ramp, list(rows))


@pytest.mark.parametrize("workers", [1, 2, 4])
@pytest.mark.parametrize("mode", [1, 6])
def test_cs_table(ob, pipes, workers, mode):
    t = cs_table(mode)
    for gcols in ([1, 2], [4, 1, 2]):
        got = pipes[workers].group_by(t.image, None, gcols, AGGS, blocks_per_batch=3, ramp=2)
        assert_model(got, t, gcols, AGGS, range(t.n), (workers, gcols))


def test_pax_table_with_cs_layout(ob, pipes):
    t = cs_table(1, pax=True)
    got = pipes[4].group_by(t.image, ob.White(0, ob.WHITE_OP_GE, (t.n // 3,)), [1, 2], AGGS, blocks_per_batch=2)
    assert_model(got, t, [1, 2], AGGS, [r for r in range(t.n) if t.cells[0][r] >= t.n // 3])


# ---- stored blocks, zero copy, skip index ---------------------------------------------------------------------------------
@pytest.mark.parametrize("comp", ["lz4", "zstd", "zlib"])
def test_stored_blocks(ob, pipes, comp):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    c = {"lz4": ob.capi.COMPRESSOR_LZ4, "zstd": ob.capi.COMPRESSOR_ZSTD_1_3_8, "zlib": ob.capi.COMPRESSOR_ZLIB}[comp]
    stored = compress_table(t.image, c)
    got = pipes[2].group_by(stored, None, [2, 1], STR_AGGS, blocks_per_batch=4, compressor=c)
    assert_model(got, t, [2, 1], STR_AGGS, range(t.n), comp)
    assert got[2].h2d_bytes == stored.image.size


def test_zero_copy_pinned_image(ob, pipes):
    import torch
    t = string_table()
    pinned = torch.empty(t.image.image.size + 256, dtype=torch.uint8).pin_memory()
    img = pinned.numpy()
    img[:t.image.image.size] = t.image.image
    img[t.image.image.size:] = 0
    table = ob.TableImage(img[:t.image.image.size], t.image.offsets, t.image.sizes, t.image.total_rows, t.image.n_cols)
    got = pipes[4].group_by(table, None, [1, 2], STR_AGGS, blocks_per_batch=3, zero_copy=True)
    stats = assert_model(got, t, [1, 2], STR_AGGS, range(t.n))
    assert_stats(stats, table, 3, 0, list(range(t.n)), zero_copy=True)


def test_skip_index_pruned_blocks(ob, pipes):
    table, agg, truth, blocks = path_table(ob, 133)
    cells = path_cells(ob, 133)
    n = PATH_ROWS[133]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    flt = ob.White(0, ob.WHITE_OP_BT, (lo, hi))
    rows = [i for i in range(n) if lo <= i <= hi]

    class T:
        pass
    t = T()
    t.cells = cells
    for gcols in ([2, 3], [4, 2]):
        got = pipes[2].group_by(table, flt, gcols, PATH_AGGS[1], blocks_per_batch=5, agg_rows=agg[0], agg_off=agg[1])
        assert_model(got, t, gcols, PATH_AGGS[1], rows, gcols)
        assert_stats(got[2], table, 5, 0, rows)


# ---- workers at once on the shared fold, each batch with its own shared-memory size ---------------------------------------
@pytest.mark.parametrize("workers", [2, 4])
@pytest.mark.parametrize("bpb", [1, 2])
def test_workers_with_different_shared_fold_sizes(ob, pipes, workers, bpb):
    class T:
        pass
    t = T()
    t.cells = vary_cells()
    aggs = [(COUNT, -1), (SUM, 0), (MAX, 0)]
    for gcols in ([1, 2], [2, 1]):
        got = pipes[workers].group_by(vary_table(), None, gcols, aggs, blocks_per_batch=bpb)
        assert_model(got, t, gcols, aggs, range(len(t.cells[0])), (workers, bpb, gcols))


# ---- the 65 536-value cap applies per batch -------------------------------------------------------------------------------
def test_value_cap_is_per_batch(ob, pipes):
    table = cap_split_table()
    cells = cap_split_cells()

    class T:
        pass
    t = T()
    t.cells = cells
    aggs = [(COUNT, -1), (SUM, 0), (MIN, 0), (MAX, 0)]
    p = pipes[4]
    got = p.group_by(table, None, [1], aggs, blocks_per_batch=CAP_SPLIT)     # every batch under the cap, the table over it
    keys, out, stats = got
    assert len(keys) > 65536
    assert_model(got, t, [1], aggs, range(len(cells[0])))
    with pytest.raises(ob.ObGpuError) as e:                                  # one batch of the whole table: over the cap
        p.group_by(table, None, [1], aggs, blocks_per_batch=table.n_blocks)
    assert e.value.code == ob.OB_NOT_SUPPORTED and "65536" in str(e.value)
    again = p.group_by(table, None, [1], aggs, blocks_per_batch=CAP_SPLIT)    # the pipeline stays usable
    assert again[0] == keys and np.array_equal(again[1], out)


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_refusals(ob, pipes):
    a = auto_table()
    p = pipes[2]
    for gcols in ([1, 3], [3, 1]):                                            # OBGPU_ENC_AUTO columns with RAW blocks
        with pytest.raises(ob.ObGpuError) as e:
            p.group_by(a.image, None, gcols, [(COUNT, -1)], blocks_per_batch=2)
        assert e.value.code == ob.OB_NOT_SUPPORTED and "dictionary" in str(e.value)
    # row output, row ids, block tables or scalar aggregates: the call returns groups only
    lib = ob.capi.lib
    t = string_table()
    spec, keep = p._spec(t.image, None, [0], 3, 1.0, 0, 0, None, None)
    res = ob.capi.HostScanResult()
    rows = np.zeros(64, dtype=np.int64)
    res.batch_row_begin, res.batch_rows, res.n_batches_cap = rows.ctypes.data, rows.ctypes.data, 64
    cols = np.array([1, 2], dtype=np.int32)
    aggs = np.array([(COUNT, -1)], dtype=np.int32)
    ids = np.zeros(t.n, dtype=np.int32)
    hagg = (ob.capi.HostAgg * 1)()
    h = C.c_void_p()

    def call():
        return lib.obgpu_pipeline_group_by(p._h, C.byref(spec), cols.ctypes.data, 2, aggs.ctypes.data, 1, C.byref(res), C.byref(h))
    spec.no_row_output = 0
    assert call() == ob.OB_INVALID_ARGUMENT and not h.value
    spec.no_row_output = 1
    spec.out_row_ids = ids.ctypes.data
    assert call() == ob.OB_INVALID_ARGUMENT
    spec.out_row_ids = None
    spec.aggs, spec.n_aggs = hagg, 1
    assert call() == ob.OB_INVALID_ARGUMENT
    spec.n_aggs = 0
    assert call() == ob.OB_SUCCESS and h.value
    lib.obgpu_groups_free(h)
    got = p.group_by(t.image, None, [2, 1], STR_AGGS, blocks_per_batch=3)     # still usable
    assert_model(got, t, [2, 1], STR_AGGS, range(t.n))
