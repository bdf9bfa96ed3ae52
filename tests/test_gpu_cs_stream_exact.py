"""CS integer streams decoded at batch open (stream_codecs.cuh) against the values that were written: the tables of
tests/test_cs_stream_exact.py (every codec, stored width, stream kind and block size; the census there shows they reach every
decoder path), not the oracle.

Per batch: the restated image read back from the device equals the oracle's restatement block for block (128-byte slots), and
scans with and without the pipelined small-block kernels (OBGPU_PIPE=1 / 0) return exactly the written values. Column-matrix
tables also run a BT over the middle half of every integer column, an NU leaf, and an EQ leaf per string column, so the filter
kernels read the restated streams too; string pointers still address the caller's coded image. The table whose restatement
needs four-byte END offsets and the one crossing to two-byte ones are checked from the read-back bytes; one coded table is
opened from a host image, from a device image without a host view, as LZ4-stored blocks and as macro blocks."""
import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import oracle_value
from test_cs_stream_codecs import MODES
from test_cs_stream_exact import (COLUMN_TABLES, GROUPS, ROWS, WIDTHS, block_starts, column_filters, column_spec, column_table,
                                  offsets_width_tag, selected_rows, stream_matrix, widening_table)

pytestmark = pytest.mark.gpu

MAX_PROJ = 24        # kMaxProj: columns one scan projects


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def device_bytes(batch):
    """the batch's device image, gathered by torch through the CUDA array interface"""
    import torch
    base, size = batch.device_image()

    class DeviceBytes:
        __cuda_array_interface__ = {"shape": (size,), "typestr": "|u1", "data": (base, False), "version": 3}
    return torch.as_tensor(DeviceBytes(), device="cuda").cpu().numpy()


def check_restated_image(batch, table):
    """block i of the device image sits at the prefix sum of the restated sizes rounded up to 128 (slot_layout) and equals
    ora.cs_transform of the coded block from header_size on; the rest of its slot is zero"""
    img = device_bytes(batch)
    pos = 0
    for i in range(table.n_blocks):
        blk = table.block(i)
        hs = int(blk[4:8].view(np.uint32)[0])
        want = ora.cs_transform(blk)
        slot = (want.size + 127) // 128 * 128
        assert np.array_equal(img[pos + hs:pos + want.size], want[hs:]), i
        assert not img[pos + want.size:pos + slot].any(), i
        pos += slot
    assert img.size == pos
    return img


def projected_ints(res, k, obj):
    data, _, nulls = res.fetch_col(k)
    j = np.arange(len(data))
    isnull = ((nulls[j // 64] >> (j % 64).astype(np.uint64)) & np.uint64(1)).tolist()
    return [None if z else oracle_value(obj, v) for v, z in zip(data.tolist(), isnull)]


def projected_strings(res, k):
    _, _, nulls = res.fetch_col(k)
    heap, off = res.fetch_strings(k)
    return [None if (int(nulls[j // 64]) >> (j % 64)) & 1 else bytes(heap[off[j]:off[j + 1]]) for j in range(len(off) - 1)]


def every_row(table):
    return np.concatenate([np.arange(r, dtype=np.int32) for r in np.diff(block_starts(table))])


# ---- 1. the stream matrix ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ub", sorted(WIDTHS))
@pytest.mark.parametrize("mode", sorted(MODES))
def test_stream_matrix_restates_and_scans_exactly(ob, ctx, monkeypatch, mode, ub):
    table, _, values = stream_matrix(mode, ub)
    n_cols = len(values[0])
    batch = ctx.open_batch(table)
    try:
        check_restated_image(batch, table)
        for pipe in ("1", "0"):
            monkeypatch.setenv("OBGPU_PIPE", pipe)
            res = batch.scan(None, list(range(n_cols)), want_row_ids=True)
            assert res.selected_rows == table.total_rows
            assert np.array_equal(res.fetch_row_ids(), every_row(table))
            for c in range(n_cols):
                data, _, nulls = res.fetch_col(c)
                assert not nulls.any() and np.array_equal(data, np.concatenate([v[c] for v in values])), (MODES[mode], ub, pipe, c)
            res.free()
    finally:
        batch.close()


# ---- 2. the column matrix ----------------------------------------------------------------------------------------------------
def check_column_scans(batch, spec, table, pipes, monkeypatch):
    starts = block_starts(table)
    for pipe in pipes:
        monkeypatch.setenv("OBGPU_PIPE", pipe)
        for lo in range(0, len(spec.cols), MAX_PROJ):
            proj = list(range(lo, min(lo + MAX_PROJ, len(spec.cols))))
            res = batch.scan(None, proj, want_row_ids=True)
            assert res.selected_rows == spec.n
            assert np.array_equal(res.fetch_row_ids(), every_row(table))
            for k, c in enumerate(proj):
                got = projected_strings(res, k) if spec.is_str(c) else projected_ints(res, k, spec.obj[c])
                assert got == spec.truth[c], (pipe, spec.names[c])
            res.free()
        for c, f, want in column_filters(spec):
            res = batch.scan(f, [c], want_row_ids=True)
            assert selected_rows(starts, res.fetch_sel_offsets(), res.fetch_row_ids()) == want, (pipe, spec.names[c], f)
            res.free()


@pytest.mark.parametrize("mode,rpb", COLUMN_TABLES)
@pytest.mark.parametrize("group", GROUPS)
def test_column_matrix_scans_and_filters_exactly(ob, ctx, monkeypatch, mode, rpb, group):
    spec = column_spec(group, ROWS[rpb])
    table = column_table(mode, rpb, group)
    batch = ctx.open_batch(table)
    try:
        check_restated_image(batch, table)
        check_column_scans(batch, spec, table, ("1", "0"), monkeypatch)
        if group == "dict_str":
            # pointers of a var-length CS_STRING column address the caller's coded image (XformRec.str_delta)
            c = spec.names.index(("string", "mid", "n0"))
            base = 0x20_0000_0000
            res = batch.scan(None, [c], string_base=base)
            ptrs, lens, _ = res.fetch_col(0)
            got = [bytes(table.image[int(p) - base:int(p) - base + int(n)]) for p, n in zip(ptrs.tolist(), lens.tolist())]
            assert got == spec.truth[c]
            res.free()
    finally:
        batch.close()


# ---- 3. END offsets the restatement widens; open paths -------------------------------------------------------------------------
@pytest.mark.parametrize("which,tag", [("four", 2), ("two", 1)])
def test_restated_end_offsets_widen(ob, ctx, monkeypatch, which, tag):
    table, _, spec = widening_table(which)
    batch = ctx.open_batch(table)
    try:
        img = check_restated_image(batch, table)
        size = ora.cs_transform(table.block(0)).size
        assert offsets_width_tag(img[:size]) == tag and offsets_width_tag(table.block(0)) == tag - 1
        check_column_scans(batch, spec, table, ("1", "0"), monkeypatch)
    finally:
        batch.close()


def test_open_paths_scan_alike(ob, ctx, monkeypatch):
    import torch
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    spec = column_spec("dict_str", ROWS[129])
    table = column_table(0, 129, "dict_str")
    dev = torch.from_numpy(table.image).cuda()
    torch.cuda.synchronize()
    stored = compress_table(table, 2)
    assert (stored.sizes < table.sizes).any()
    macro = build_macro_blocks(table, spec.obj, 1)
    batches = {"host": ctx.open_batch(table),
               "device": ob.PageBatch(ctx, table, device_image_ptr=dev.data_ptr(), image_size=table.image.size, host_view=False),
               "lz4": ob.PageBatch(ctx, stored, compressor=2),
               "macro": ob.PageBatch.from_macro_blocks(ctx, macro.image, macro.macro_block_size, macro.n_macro)}
    try:
        for name, batch in batches.items():
            assert batch.n_blocks == table.n_blocks, name
            check_column_scans(batch, spec, table, ("0",), monkeypatch)
    finally:
        for batch in batches.values():
            batch.close()
