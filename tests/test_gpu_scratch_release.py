"""Refusals release their device scratch. Each entry point below is driven into a refusal that malformed or undersized input
reaches, most of them after the call has allocated device memory. The call returns its code, and once the ctx stream is
synchronised the device's default memory pool (where the library allocates, stream-ordered) is back to the bytes in use before
the call: nothing allocated on the way to the refusal is left behind. The same ctx then completes a normal scan."""
import ctypes as C

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_gpu_agg_rows import _raw as _agg_rows_call, upload
from test_gpu_device_compress import _frame, _on_device, _raw_call as _compress_call, payload_shapes
from test_gpu_lz4_blocks import _table
from test_gpu_macro_blocks import make_table as make_macro_table
from test_gpu_pipeline_compressed import _tables as string_tables

pytestmark = pytest.mark.gpu
LZ4, ZLIB, ZSTD = 2, 4, 6
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7


def _pool_used():
    """Bytes in use from device 0's default memory pool (its release threshold is UINT64_MAX, so this is exact)."""
    cu = C.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def env(ob):
    ctx = ob.ScanContext(0)
    table, _ = _table(n=9000)
    plain = ob.PageBatch(ctx, table)
    yield ctx, table, plain
    plain.close()
    ctx.close()


def _code(ob, fn):
    """fn's OB code: 0 when it returns, the ObGpuError's code when it raises."""
    try:
        out = fn()
    except ob.ObGpuError as e:
        return e.code
    if hasattr(out, "close"):
        out.close()
    return out if isinstance(out, int) else 0


def _refused(ob, env, fn, code):
    ctx, table, plain = env
    ctx.synchronize()
    before = _pool_used()
    assert _code(ob, fn) == code
    ctx.synchronize()
    assert _pool_used() == before
    r = plain.scan(None, [0, 1])
    assert r.selected_rows == table.total_rows
    r.free()


def _reopen(ob, ctx, st, image, compressor):
    return lambda: ob.PageBatch(ctx, type(st)(image, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=compressor)


@pytest.mark.parametrize("compressor", [LZ4, ZSTD, ZLIB])
def test_stored_block_with_a_flipped_payload_byte(ob, env, compressor):
    from oceanbase_b200.sstable import compress_table
    ctx, table, _ = env
    st = compress_table(table, compressor)
    hs, ln, zl = lz4_ref.header_fields(st.block(3))
    assert zl < ln
    bad = st.image.copy()
    bad[st.offsets[3] + hs + zl // 2] ^= 0x20
    _refused(ob, env, _reopen(ob, ctx, st, bad, compressor), ob.OB_INVALID_DATA)
    assert "checksum" in ctx.last_error()


def test_malformed_zstd_frame_under_a_correct_checksum(ob, env):
    from oceanbase_b200.sstable import compress_table
    ctx, table, _ = env
    st = compress_table(table, ZSTD)
    crc = lambda a: int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))
    hs, ln, zl = lz4_ref.header_fields(st.block(3))
    bad = st.image.copy()
    b = bad[st.offsets[3]:st.offsets[3] + st.sizes[3]]
    pay = b[hs:]
    assert pay[4] & 0x20 and (pay[4] >> 6) == 1   # Single_Segment, 2-byte Frame_Content_Size: one more than data_length_
    v = int(pay[5]) | (int(pay[6]) << 8)
    pay[5], pay[6] = (v + 1) & 0xff, (v + 1) >> 8
    b[48:56] = np.frombuffer(np.uint64(crc(np.ascontiguousarray(pay))).tobytes(), np.uint8)
    b[8:10] = 0
    b[8:10] = np.frombuffer(np.uint16(lz4_ref.header_checksum_fold(b)).tobytes(), np.uint8)
    assert lz4_ref.stored_checksums_ok(b, crc)
    _refused(ob, env, _reopen(ob, ctx, st, bad, ZSTD), ob.OB_INVALID_DATA)
    assert "zstd" in ctx.last_error()


def test_macro_block_with_a_bad_header(ob, env):
    from oceanbase_b200.sstable import build_macro_blocks
    ctx = env[0]
    table, types = make_macro_table(n=30_000)
    mi = build_macro_blocks(table, types, 1, macro_block_size=128 << 10)
    bad = mi.image.copy()
    bad[8] = 0x55   # common header magic
    _refused(ob, env, lambda: ob.PageBatch.from_macro_blocks(ctx, bad, 128 << 10, mi.n_macro), ob.OB_INVALID_DATA)


def test_cs_block_with_a_corrupt_stream_layout(ob, env):
    from oceanbase_b200.sstable import TableImage
    ctx = env[0]
    st = string_tables(ob)["cs"][0]
    bad = st.image.copy()
    o = int(st.offsets[2])
    header_size = int(bad[o + 4:o + 8].view(np.uint32)[0])
    bad[o + header_size] = 1   # the CS column area's version byte
    _refused(ob, env, lambda: ob.PageBatch(ctx, TableImage(bad, st.offsets, st.sizes, st.total_rows, st.n_cols)), ob.OB_INVALID_DATA)
    assert ctx.last_error() == "corrupt CS micro block (stream layout)"


def test_agg_rows_with_out_cap_one_byte_short(ob, env):
    ctx = env[0]
    rng = np.random.default_rng(8)
    n = 5000
    dcols, keep = upload([(5, rng.integers(-9, 9, n), None), (9, rng.integers(0, 9, n), (rng.random(n) < 0.2).astype(np.uint8))])
    code, size = _agg_rows_call(ob, ctx, dcols, [0, 1], n, 100)
    assert code == ob.OB_SUCCESS and size > 0
    out = np.zeros(size, dtype=np.uint8)
    offs = np.zeros(n // 100 + 1, dtype=np.int64)
    _refused(ob, env, lambda: _agg_rows_call(ob, ctx, dcols, [0, 1], n, 100, out.ctypes.data, size - 1, offs.ctypes.data)[0],
             ob.OB_BUF_NOT_ENOUGH)


def test_compress_blocks_with_out_cap_one_byte_short(ob, env):
    import torch
    ctx = env[0]
    table = _frame(payload_shapes()[:20])
    img, off, sz = _on_device(table)
    code, cap = _compress_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), table.n_blocks, LZ4, 128, None, 0)
    assert code == ob.OB_SUCCESS
    out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    for comp in (LZ4, ZSTD):
        _refused(ob, env, lambda: _compress_call(ctx, img.data_ptr(), off.data_ptr(), sz.data_ptr(), table.n_blocks, comp, 128,
                                                 out.data_ptr(), cap - 1)[0], ob.OB_BUF_NOT_ENOUGH)


def test_result_strings_with_a_heap_one_byte_short(ob, env):
    from oceanbase_b200.capi import lib
    ctx = env[0]
    batch = ob.PageBatch(ctx, string_tables(ob)["pax"][0])
    res = batch.scan(None, [0, 6, 7])
    rows = res.selected_rows
    heap, _ = res.fetch_strings(1)
    assert heap.size > 1
    short = np.zeros(heap.size - 1, dtype=np.uint8)
    off = np.zeros(rows + 1, dtype=np.int64)
    need = C.c_int64(0)
    _refused(ob, env, lambda: lib.obgpu_result_fetch_strings(res._h, 1, 0, rows, short.ctypes.data, short.size, off.ctypes.data,
                                                            C.byref(need)), ob.OB_BUF_NOT_ENOUGH)
    assert need.value == heap.size
    # the heap fetch must name the rows obgpu_result_string_bytes sized
    ca = (C.c_int32 * 2)(1, 2)
    nb = np.zeros(2, dtype=np.int64)
    assert lib.obgpu_result_string_bytes(res._h, 2, ca, 0, 100, nb.ctypes.data) == 0
    heaps = [np.zeros(int(b) + 1, dtype=np.uint8) for b in nb]
    hh = (C.c_void_p * 2)(*[h.ctypes.data for h in heaps])
    _refused(ob, env, lambda: lib.obgpu_result_fetch_string_heap(res._h, 2, ca, 0, 99, hh, None), ob.OB_INVALID_ARGUMENT)
    res.free()
    batch.close()


def test_merge_result_strings_without_images(ob, env):
    import torch
    from oceanbase_b200 import compaction
    from oceanbase_b200.capi import lib
    ctx = env[0]
    n = 1000
    runs = [compaction.DecodedRun(torch.arange(r, 2 * n, 2, dtype=torch.int64, device="cuda"), None,
                                  [torch.arange(n, dtype=torch.int64, device="cuda")], [torch.zeros(n, dtype=torch.uint8, device="cuda")])
            for r in range(2)]
    res = compaction.merge_decoded(ctx, runs)
    rows = res.info().out_rows
    off = np.zeros(rows + 1, dtype=np.int64)
    nl = np.zeros(rows, dtype=np.uint8)
    heap = np.zeros(64, dtype=np.uint8)
    need = C.c_int64(0)
    _refused(ob, env, lambda: lib.obgpu_merge_result_fetch_strings(res._h, 0, 0, rows, heap.ctypes.data, heap.size, off.ctypes.data,
                                                                  nl.ctypes.data, C.byref(need)), ob.OB_INVALID_ARGUMENT)
    assert ctx.last_error() == "no page-batch images attached to the merge result"
    res.free()
