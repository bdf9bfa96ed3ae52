"""ORDER BY ... LIMIT k through the host pipeline (obgpu_pipeline_top_rows, HostScanPipeline.top_rows): the rows of every page
batch merged on the device must be byte for byte those of obgpu_result_top_rows over the whole table opened as one batch, and so
those of the plain model of test_gpu_top_rows (positions are block indexes of the table).

Sweeps: blocks per batch 1, 3, 7, all, more than all and the default; ramps 0 and 2; 1, 2 and 4 workers; no filter, a selective
filter and one that selects nothing; k from 1 past the selection; PAX and CS tables; LZ4-, zstd- and zlib-stored blocks; a
zero-copy pinned image; skip-index-pruned blocks; ties that straddle batch boundaries (an all-equal key and a 16-value key over
140 blocks); the refusals, with the pipeline usable after each."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_aggregate_exact import PATH_ROWS, path_table
from test_gpu_group_by_values import path_cells
from test_gpu_top_rows import model_order, positions
from test_scan_codes_model import auto_table, cs_table, string_table
from test_top_rows_shapes import big_table

pytestmark = pytest.mark.gpu


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


def one_batch(ctx, image, flt, keys, outs, k, **kw):
    batch = ctx.open_batch(image, **kw)
    res = batch.scan(flt, [0])
    try:
        return res.top_rows(keys, outs, k)
    finally:
        res.free()
        batch.close()


def assert_same(ctx, p, image, flt, keys, outs, k, what, open_kw=None, **kw):
    got_pos, got_rows, stats = p.top_rows(image, flt, keys, outs, k, **kw)
    want_pos, want_rows = one_batch(ctx, image, flt, keys, outs, k, **(open_kw or {}))
    assert got_pos == want_pos, what
    assert got_rows == want_rows, what
    return got_pos, got_rows, stats


STR_KEYS = [[(2, 0, 1), (1, 1, 0)], [(1, 1, 1)], [4, (2, 1, 0), 0]]


@pytest.mark.parametrize("bpb", [1, 3, 7, "all", "more", 0])
@pytest.mark.parametrize("ramp", [0, 2])
def test_batch_cuts(ob, ctx, pipes, bpb, ramp):
    t = string_table()
    n = t.image.n_blocks
    b = {"all": n, "more": n + 5}.get(bpb, bpb)
    half = t.n // 2
    filters = [(None, range(t.n)), (ob.White(0, ob.WHITE_OP_LT, (half,)), [r for r in range(t.n) if t.cells[0][r] < half]),
               (ob.White(0, ob.WHITE_OP_LT, (0,)), [])]
    batch = ctx.open_batch(t.image)
    pos = positions(batch)
    batch.close()
    for i, (flt, rows) in enumerate(filters):
        for j, keys in enumerate(STR_KEYS):
            p = pipes[(1, 2, 4)[(i + j) % 3]]
            for k in (1, 17, max(len(rows) - 1, 1), len(rows) + 3):
                got_pos, got_rows, stats = assert_same(ctx, p, t.image, flt, keys, [1, 2, 3], k, (bpb, ramp, i, keys, k),
                                                       blocks_per_batch=b, ramp=ramp)
                order = model_order(t.cells, list(rows), keys, pos)[:k]
                assert got_pos == [pos[r] for r in order] and got_rows == [(t.cells[1][r], t.cells[2][r], t.cells[3][r]) for r in order]
                assert stats.selected_rows == len(rows)


@pytest.mark.parametrize("workers", [1, 2, 4])
@pytest.mark.parametrize("mode", [1, 4])
def test_cs_table(ob, ctx, pipes, workers, mode):
    t = cs_table(mode)
    for keys in ([(3, 1, 0)], [(4, 0, 1), (1, 1, 0), 2]):
        assert_same(ctx, pipes[workers], t.image, None, keys, [4, 3, 1], 100, (workers, mode, keys), blocks_per_batch=2)


@pytest.mark.parametrize("comp", ["lz4", "zstd", "zlib"])
def test_stored_blocks(ob, ctx, pipes, comp):
    from oceanbase_b200.sstable import compress_table
    t = string_table()
    c = {"lz4": ob.capi.COMPRESSOR_LZ4, "zstd": ob.capi.COMPRESSOR_ZSTD_1_3_8, "zlib": ob.capi.COMPRESSOR_ZLIB}[comp]
    stored = compress_table(t.image, c)
    for keys in STR_KEYS:
        assert_same(ctx, pipes[2], stored, None, keys, [1, 2], 300, (comp, keys), open_kw={"compressor": c}, blocks_per_batch=4,
                    compressor=c)


def test_zero_copy_pinned_image(ob, ctx, pipes):
    import torch
    t = string_table()
    pinned = torch.empty(t.image.image.size + 256, dtype=torch.uint8).pin_memory()
    img = pinned.numpy()
    img[:t.image.image.size] = t.image.image
    img[t.image.image.size:] = 0
    table = ob.TableImage(img[:t.image.image.size], t.image.offsets, t.image.sizes, t.image.total_rows, t.image.n_cols)
    _, _, stats = assert_same(ctx, pipes[4], table, None, STR_KEYS[0], [1, 2], 500, "zero copy", blocks_per_batch=3, zero_copy=True)
    assert stats.h2d_bytes == 0


def test_skip_index_pruned_blocks(ob, ctx, pipes):
    table, agg, truth, blocks = path_table(ob, 133)
    n = PATH_ROWS[133]
    lo, hi = n // 4 + 3, 3 * n // 4 - 3
    flt = ob.White(0, ob.WHITE_OP_BT, (lo, hi))
    for keys in ([(2, 1, 0)], [(4, 0, 1), 3]):
        assert_same(ctx, pipes[2], table, flt, keys, [0, 2, 4], 250, keys, blocks_per_batch=5, agg_rows=agg[0], agg_off=agg[1])


def test_ties_across_batches(ob, ctx, pipes):
    image, cells = big_table()
    for keys, k in (([1], 65536), ([(1, 1, 0)], 3000), ([(2, 0, 0)], 65536), ([(2, 1, 1)], 1000), ([3, (2, 1, 0)], 5000)):
        for w, bpb in ((4, 7), (2, 33), (1, 0)):
            assert_same(ctx, pipes[w], image, None, keys, [0, 2, 3], k, (keys, k, w, bpb), blocks_per_batch=bpb)


def test_refusals(ob, ctx, pipes):
    p = pipes[2]
    t = string_table()
    a = auto_table()
    mixed = ob.TableImage.concat([t.image, a.image])           # column 1: VARCHAR in one part, INT in the other
    for keys, outs, code in (([1], [0], ob.OB_NOT_SUPPORTED), ([0], [1], ob.OB_NOT_SUPPORTED)):
        with pytest.raises(ob.ObGpuError) as e:
            p.top_rows(mixed, None, keys, outs, 5, blocks_per_batch=t.image.n_blocks)
        assert e.value.code == code and str(e.value)
        assert_same(ctx, p, t.image, None, STR_KEYS[0], [1], 9, "usable", blocks_per_batch=3)
    with pytest.raises(ob.ObGpuError) as e:
        p.top_rows(t.image, None, [1], [1], 65537, blocks_per_batch=3)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    for keys, outs, k in (([], [1], 5), ([1] * 5, [1], 5), ([1], [1] * 17, 5), ([1], [1], 0), ([9], [1], 5), ([1], [9], 5)):
        with pytest.raises(ob.ObGpuError) as e:
            p.top_rows(t.image, None, keys, outs, k, blocks_per_batch=3)
        assert e.value.code == ob.OB_INVALID_ARGUMENT, (keys, outs, k)
        lib = ob.capi.lib
        z = np.zeros(8, dtype=np.int64)
        assert lib.obgpu_pipeline_fetch_top_rows(p._h, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data) \
            == ob.OB_INVALID_ARGUMENT                            # a refused call leaves no rows
    # row output, row ids or scalar aggregates: the call returns rows only
    lib = ob.capi.lib
    spec, keep = p._spec(t.image, None, [0], 3, 1.0, 0, 0, None, None)
    res = ob.capi.HostScanResult()
    rows = np.zeros(64, dtype=np.int64)
    res.batch_row_begin, res.batch_rows, res.n_batches_cap = rows.ctypes.data, rows.ctypes.data, 64
    karr = np.array([[1, 0, 0]], dtype=np.int32)
    outs = np.array([1], dtype=np.int32)
    nr, hb = C.c_int64(), C.c_int64()

    def call():
        return lib.obgpu_pipeline_top_rows(p._h, C.byref(spec), karr.ctypes.data, 1, outs.ctypes.data, 1, 5, C.byref(res), C.byref(nr),
                                           C.byref(hb))
    spec.no_row_output = 0
    assert call() == ob.OB_INVALID_ARGUMENT
    spec.no_row_output = 1
    ids = np.zeros(t.n, dtype=np.int32)
    spec.out_row_ids = ids.ctypes.data
    assert call() == ob.OB_INVALID_ARGUMENT
    spec.out_row_ids = None
    assert call() == ob.OB_SUCCESS and nr.value == 5
    assert_same(ctx, p, t.image, None, STR_KEYS[2], [2, 1], 40, "usable after", blocks_per_batch=2)
