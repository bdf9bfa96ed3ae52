"""GROUP BY columns of any encoding through the host pipeline (obgpu_pipeline_group_by_any, HostScanPipeline.group_by_any):
the groups of every page batch, each grouped on the path its blocks allow and merged on the device, equal the one-batch
ScanResult.group_by_any byte for byte and the plain tuple model (test_gpu_group_by_columns.tuple_model).

Sweeps: batch sizes of 1, 3, 7, all and more than all blocks and the default; ramps 0 and 2; 1, 2 and 4 workers; auto_table
(dictionary-only batches next to batches with RAW blocks: 0 < cells_batches < n_batches) and a RAW matrix table; LZ4-, zstd- and
zlib-stored blocks; a zero-copy pinned image; skip-index-pruned blocks; cap_table as one batch, which obgpu_pipeline_group_by
refuses; the spec refusals."""
import numpy as np
import pytest

from test_aggregate_exact import COUNT, MAX, MIN, SUM, K, M, VA, VB, W, matrix_spec, matrix_table
from test_gpu_aggregate_exact import PATH_AGGS, PATH_ROWS, path_table
from test_gpu_group_by_columns import tuple_model
from test_gpu_group_by_values import path_cells
from test_gpu_pipeline_group_by import assert_stats
from test_scan_codes_model import CAP, auto_table, cap_table

pytestmark = pytest.mark.gpu

AUTO_AGGS = [(COUNT, -1), (SUM, 0), (MIN, 3), (MAX, 1), (COUNT, 1)]
RAW_AGGS = [(COUNT, -1), (SUM, VA), (MIN, VB), (MAX, W), (COUNT, VB)]


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pipes():
    from oceanbase_b200.pipeline import HostScanPipeline
    ps = {w: HostScanPipeline(0, n_workers=w) for w in (1, 2, 4)}
    yield ps
    for p in ps.values():
        p.close()


def one_batch(ctx, image, flt, gcols, aggs, **kw):
    batch = ctx.open_batch(image, **kw)
    res = batch.scan(flt, [0])
    keys, out, _ = res.group_by_any(gcols, aggs)
    res.free()
    batch.close()
    return keys, out


def check(got, want, cells, gcols, aggs, rows, what):
    keys, out, stats, cells_batches = got
    assert keys == want[0] and out.tobytes() == want[1].tobytes(), what
    mk, mout = tuple_model([cells[c] for c in gcols], list(rows), aggs, cells)
    assert keys == mk and np.array_equal(out, mout), what
    assert 0 <= cells_batches <= stats.n_batches
    return stats, cells_batches


@pytest.mark.parametrize("bpb", [1, 3, 7, "all", "more", 0])
@pytest.mark.parametrize("ramp", [0, 2])
def test_batch_cuts(ob, ctx, pipes, bpb, ramp):
    t = auto_table()
    spec = matrix_spec("int", "raw")
    raw = matrix_table("int", "raw")
    for i, (image, cells, n, keysets, aggs) in enumerate(((t.image, t.cells, t.n, ([1], [2, 1], [1, 2, 3]), AUTO_AGGS),
                                                          (raw, spec.truth, spec.n, ([VA], [VB, M], [W, VA]), RAW_AGGS))):
        nb = image.n_blocks
        b = {"all": nb, "more": nb + 5}.get(bpb, bpb)
        half = n // 2
        for j, (flt, rows) in enumerate(((None, range(n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), range(half)))):
            for gcols in keysets:
                p = pipes[(1, 2, 4)[(i + j + len(gcols)) % 3]]
                got = p.group_by_any(image, flt, gcols, aggs, blocks_per_batch=b, ramp=ramp)
                stats, _ = check(got, one_batch(ctx, image, flt, gcols, aggs), cells, gcols, aggs, rows, (bpb, ramp, gcols, j))
                assert_stats(stats, image, b, ramp, list(rows))


def test_mixed_paths(pipes):
    """auto_table cut into batches of 3 blocks: the first holds only dictionary-coded blocks, the others a RAW block each"""
    t = auto_table()
    for w in (1, 2, 4):
        keys, out, stats, cells_batches = pipes[w].group_by_any(t.image, None, [1], AUTO_AGGS, blocks_per_batch=3)
        assert stats.n_batches == 4 and cells_batches == 3, (w, cells_batches)
        mk, mout = tuple_model([t.cells[1]], range(t.n), AUTO_AGGS, t.cells)
        assert keys == mk and np.array_equal(out, mout)


@pytest.mark.parametrize("comp", ["COMPRESSOR_LZ4", "COMPRESSOR_ZSTD_1_3_8", "COMPRESSOR_ZLIB"])
def test_stored_blocks(ob, ctx, pipes, comp):
    from oceanbase_b200.sstable import compress_table
    c = getattr(ob.capi, comp)
    t = auto_table()
    stored = compress_table(t.image, c)
    for gcols in ([2], [1, 2, 3]):
        got = pipes[2].group_by_any(stored, None, gcols, AUTO_AGGS, blocks_per_batch=5, compressor=c)
        check(got, one_batch(ctx, t.image, None, gcols, AUTO_AGGS), t.cells, gcols, AUTO_AGGS, range(t.n), (comp, gcols))


def test_zero_copy_pinned_image(ob, ctx, pipes):
    import torch
    t = auto_table()
    pinned = torch.empty(t.image.image.size + 256, dtype=torch.uint8).pin_memory()
    img = pinned.numpy()
    img[:t.image.image.size] = t.image.image
    img[t.image.image.size:] = 0
    table = ob.TableImage(img[:t.image.image.size], t.image.offsets, t.image.sizes, t.image.total_rows, t.image.n_cols)
    got = pipes[4].group_by_any(table, None, [1, 2], AUTO_AGGS, blocks_per_batch=3, zero_copy=True)
    stats, cb = check(got, one_batch(ctx, t.image, None, [1, 2], AUTO_AGGS), t.cells, [1, 2], AUTO_AGGS, range(t.n), "zero copy")
    assert_stats(stats, table, 3, 0, list(range(t.n)), zero_copy=True)
    assert cb == 3


def test_skip_index(ob, ctx, pipes):
    table, agg, truth, blocks = path_table(ob, 133)
    cells = path_cells(ob, 133)
    n = PATH_ROWS[133]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    flt = ob.White(0, ob.WHITE_OP_BT, (lo, hi))
    rows = [i for i in range(n) if lo <= i <= hi]
    for gcols in ([0], [2, 0]):
        got = pipes[2].group_by_any(table, flt, gcols, PATH_AGGS[1], blocks_per_batch=5, agg_rows=agg[0], agg_off=agg[1])
        stats, cb = check(got, one_batch(ctx, table, flt, gcols, PATH_AGGS[1]), cells, gcols, PATH_AGGS[1], rows, gcols)
        assert cb > 0


def test_cap_table_as_one_batch(ob, ctx, pipes):
    t = cap_table()
    nb = t.image.n_blocks
    aggs = [(COUNT, -1), (SUM, 0)]
    with pytest.raises(ob.ObGpuError) as e:
        pipes[1].group_by(t.image, None, [2], aggs, blocks_per_batch=nb)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    keys, out, stats, cb = pipes[1].group_by_any(t.image, None, [2], aggs, blocks_per_batch=nb)
    assert len(keys) == CAP + 1 and stats.n_batches == 1 and cb == 1
    mk, mout = tuple_model([t.cells[2]], range(t.n), aggs, t.cells)
    assert keys == mk and np.array_equal(out, mout)


def test_spec_refusals(ob, pipes):
    import ctypes as C
    from oceanbase_b200 import capi
    t = auto_table()
    p = pipes[2]
    with pytest.raises(ob.ObGpuError) as e:
        p.group_by_any(t.image, None, [1], [(capi.AGG_SUM_PRODUCT, 0)])
    assert e.value.code == ob.OB_NOT_SUPPORTED
    for gcols in ([], [1, 2, 3, 0, 1], [9]):
        with pytest.raises(ob.ObGpuError):
            p.group_by_any(t.image, None, gcols, AUTO_AGGS)
    spec, keep = p._spec(t.image, None, [0], 3, 1.0, 0, 0, None, None)   # row output asked for
    res = capi.HostScanResult()
    rows = np.zeros(16, dtype=np.int64)
    res.batch_row_begin, res.batch_rows, res.n_batches_cap = rows.ctypes.data, rows.ctypes.data, 8
    cols = np.array([1], dtype=np.int32)
    gspec = np.array([(COUNT, -1)], dtype=np.int32)
    h, cb = C.c_void_p(), C.c_int32(7)
    assert capi.lib.obgpu_pipeline_group_by_any(p._h, C.byref(spec), cols.ctypes.data, 1, gspec.ctypes.data, 1, C.byref(res), C.byref(h),
                                                C.byref(cb)) == capi.OB_INVALID_ARGUMENT
    assert not h.value
    keys, out, stats, cells_batches = p.group_by_any(t.image, None, [1], AUTO_AGGS, blocks_per_batch=3)   # still usable
    assert cells_batches == 3
