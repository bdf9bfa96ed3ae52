"""zlib-compressed micro-blocks (compressor 4) decoded on the device: obgpu_zlib_decompress on every committed zlib stream and on
the malformed streams (the device's verdict is zlib's, or stricter only where the vectors say so); page batches opened from
compressor-4 blocks made by the writer and by the system zlib, and from compressor-4 macro blocks, scan bit for bit like the
plain batch; mixed LZ4 / zlib macro images are refused; corrupt input is refused with OBGPU_INVALID_DATA and the ctx keeps
working; string pointers rebased on obgpu_batch_device_image address the right device bytes."""
import ctypes as C
import hashlib
import zlib

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_gpu_lz4_blocks import _reframe_with, _table, scans_equal
from test_zlib_blocks import vectors

pytestmark = pytest.mark.gpu
ZLIB = 4


def _decompress(ctx, streams, out_lens):
    import torch
    from oceanbase_b200.capi import lib
    in_len = np.array([len(s) for s in streams], dtype=np.int64)
    in_off = np.concatenate([[0], np.cumsum(in_len)[:-1]]).astype(np.int64)
    out_len = np.array(out_lens, dtype=np.int64)
    out_off = np.concatenate([[0], np.cumsum(out_len)[:-1]]).astype(np.int64)
    d_in = torch.from_numpy(np.frombuffer(b"".join(streams) + b"\0", dtype=np.uint8).copy()).cuda()
    d_out = torch.zeros(int(out_len.sum()) + 1, dtype=torch.uint8, device="cuda")
    status = np.full(len(streams), -1, dtype=np.int32)
    code = lib.obgpu_zlib_decompress(ctx._h, C.c_void_p(d_in.data_ptr()), in_off.ctypes.data, in_len.ctypes.data,
                                     C.c_void_p(d_out.data_ptr()), out_off.ctypes.data, out_len.ctypes.data, len(streams), status.ctypes.data)
    out = d_out.cpu().numpy()
    return code, status, [out[o:o + n].tobytes() for o, n in zip(out_off, out_len)]


def test_zlib_decompress_golden_streams_and_malformed_streams():
    import oceanbase_b200 as ob
    streams, bad, _, _ = vectors()
    ctx = ob.ScanContext(0)
    code, status, outs = _decompress(ctx, [s for s, _ in streams], [len(p) for _, p in streams])
    assert code == 0 and (status == 0).all(), np.nonzero(status)[0]
    for (_, p), o in zip(streams, outs):
        assert o == p
    code, status, outs = _decompress(ctx, [s for s, *_ in bad], [n for _, n, *_ in bad])
    assert code == ob.OB_INVALID_DATA
    stricter = set()
    for k, ((s, n, lib_ok, digest, refusal, strict), st, o) in enumerate(zip(bad, status, outs)):
        if st == 0:   # the device accepts only what zlib accepts, with zlib's bytes
            assert lib_ok, (k, refusal)
            assert hashlib.sha256(o).digest() == digest, k
        elif lib_ok:  # stricter than zlib only where the vectors name it
            assert strict, (k, refusal)
            stricter.add(strict)
        if refusal and refusal != "trailing_bytes":
            assert st != 0, (k, refusal)
    assert stricter == {"trailing_bytes"}
    # the ctx keeps working: the golden streams decode again
    code, status, _ = _decompress(ctx, [s for s, _ in streams[:20]], [len(p) for _, p in streams[:20]])
    assert code == 0 and (status == 0).all()
    ctx.close()


@pytest.mark.parametrize("cs", [False, True])
@pytest.mark.parametrize("source,on_device", [("writer", False), ("writer", True), ("z1", False), ("z6", True), ("z6", False)])
def test_zlib_batch_scans_like_the_plain_batch(cs, source, on_device):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(cs=cs, n=20_000 if source != "writer" else 60_000)
    if source == "writer":
        st = compress_table(table, ZLIB)
    else:
        st = _reframe_with(table, lambda p: zlib.compress(bytes(p), int(source[1:])))
    n_comp = sum(1 for i in range(st.n_blocks) if lz4_ref.header_fields(st.block(i))[2] < lz4_ref.header_fields(st.block(i))[1])
    assert n_comp >= 0.9 * st.n_blocks
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    keep = None
    if on_device:
        keep = torch.from_numpy(st.image).cuda()
        cb = ob.PageBatch(ctx, st, device_image_ptr=keep.data_ptr(), image_size=st.image.size, compressor=ZLIB)
    else:
        cb = ob.PageBatch(ctx, st, compressor=ZLIB)
    assert cb.n_blocks == table.n_blocks and cb.total_rows == table.total_rows
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_mixed_blocks_and_edge_sizes():
    """Raw and compressed blocks in one batch, a 1-row block, a block above 64 KiB and one above 1 MiB."""
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, TableImage, compress_table, encode_table
    rng = np.random.default_rng(9)
    t1, _ = _table(n=9000, rpb=900)
    noise = encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(-(1 << 62), 1 << 62, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 40, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_INT, capi.ENC_DICT, rng.integers(0, 40, size=2700, dtype=np.int64)),
                          Column(capi.OBJ_VARCHAR, capi.ENC_RAW, [rng.bytes(12) for _ in range(2700)])], 900, rowkey_cnt=1)
    one, _ = _table(n=1, rpb=1)
    mid, _ = _table(n=6000, rpb=6000)
    wide = [(b"name-%04d;" % (i % 211)) * 36 for i in range(3000)]   # a 1.2 MB block of 3000 rows (a block holds <= 65535 rows)
    big = encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, np.arange(3000, dtype=np.int64) * 2 + 1),
                        Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(0, 40, size=3000, dtype=np.int64)),
                        Column(capi.OBJ_INT, capi.ENC_DICT, rng.integers(0, 40, size=3000, dtype=np.int64)),
                        Column(capi.OBJ_VARCHAR, capi.ENC_RAW, wide)], 3000, rowkey_cnt=1)
    assert mid.sizes.max() > 64 << 10 and big.sizes.max() > 1 << 20
    table = TableImage.concat([t1, noise, one, mid, big])
    st = compress_table(table, ZLIB)
    # every third block is put back in its plain (raw stored) form
    blocks = [table.block(i) if i % 3 == 1 else st.block(i) for i in range(st.n_blocks)]
    offs = np.concatenate([[0], np.cumsum([len(x) for x in blocks])[:-1]]).astype(np.int64)
    st = TableImage(np.concatenate(blocks), offs, np.array([len(x) for x in blocks], dtype=np.int64), table.total_rows, table.n_cols)
    kinds = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
    assert any(z == l for _, l, z in kinds) and any(z < l for _, l, z in kinds)
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    cb = ob.PageBatch(ctx, st, compressor=ZLIB)
    scans_equal(plain, cb)
    cb.close()
    with pytest.raises(ob.ObGpuError) as e:   # an LZ4 open of zlib payloads fails on the stream, not on the checksum
        ob.PageBatch(ctx, st, compressor=capi.COMPRESSOR_LZ4)
    assert e.value.code == ob.OB_INVALID_DATA
    plain.close()
    ctx.close()


def test_twenty_thousand_block_batch():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=20_000 * 40, rpb=40, seed=4)
    assert table.n_blocks >= 20_000
    st = compress_table(table, ZLIB)
    ctx = ob.ScanContext(0)
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=ZLIB)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


@pytest.mark.parametrize("macro_size,on_device", [(2 << 20, False), (64 << 10, True)])
def test_zlib_macro_blocks_scan_like_the_plain_image(macro_size, on_device):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import build_macro_blocks
    for cs in (False, True):
        table, types = _table(cs=cs)
        mi = build_macro_blocks(table, types, 1, macro_block_size=macro_size, compressor=ZLIB)
        ctx = ob.ScanContext(0)
        plain = ob.PageBatch(ctx, table)
        keep = None
        if on_device:
            keep = torch.from_numpy(mi.image).cuda()
            mb = ob.PageBatch.from_macro_blocks(ctx, None, macro_size, mi.n_macro, device_ptr=keep.data_ptr())
        else:
            mb = ob.PageBatch.from_macro_blocks(ctx, mi.image, macro_size, mi.n_macro)
        assert mb.n_blocks == table.n_blocks and mb.total_rows == table.total_rows
        scans_equal(plain, mb)
        mb.close()
        plain.close()
        ctx.close()


def test_macro_image_mixing_lz4_and_zlib_is_refused():
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks
    ms = 64 << 10
    table, types = _table(n=9000)
    a = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=capi.COMPRESSOR_LZ4)
    b = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=ZLIB)
    img = np.concatenate([a.image[:a.n_macro * ms], b.image[:b.n_macro * ms]])
    ctx = ob.ScanContext(0)
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch.from_macro_blocks(ctx, img, ms, a.n_macro + b.n_macro)
    assert e.value.code == ob.OB_NOT_SUPPORTED
    mb = ob.PageBatch.from_macro_blocks(ctx, b.image, ms, b.n_macro)   # the ctx keeps working
    plain = ob.PageBatch(ctx, table)
    scans_equal(plain, mb)
    mb.close()
    plain.close()
    ctx.close()


def _refit(b, hs, pay, crc):
    """Block b with payload `pay` (same length) and its payload and header checksums made right."""
    b[hs:] = pay
    b[48:56] = np.frombuffer(np.uint64(crc(np.ascontiguousarray(pay))).tobytes(), np.uint8)
    b[8:10] = 0
    b[8:10] = np.frombuffer(np.uint16(lz4_ref.header_checksum_fold(b)).tobytes(), np.uint8)


def test_corrupt_input_is_refused_and_the_ctx_keeps_working():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, ZLIB)
    crc = lambda a: int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))
    hs, ln, zl = lz4_ref.header_fields(st.block(3))
    assert zl < ln
    ctx = ob.ScanContext(0)
    reopen = lambda img: ob.PageBatch(ctx, type(st)(img, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=ZLIB)
    # a flipped header byte and a flipped payload byte: the checksums refuse them
    for at in (st.offsets[3] + 16, st.offsets[3] + hs + zl // 2):
        bad = st.image.copy()
        bad[at] ^= 0x20
        with pytest.raises(ob.ObGpuError) as e:
            reopen(bad)
        assert e.value.code == ob.OB_INVALID_DATA and "checksum" in ctx.last_error()
    # under correct checksums: a wrong Adler-32, and a stream one byte short (data_zlength_ follows)
    for what in ("adler", "truncated"):
        blocks = [st.block(i).copy() for i in range(st.n_blocks)]
        pay = blocks[3][hs:].copy()
        if what == "adler":
            pay[-1] ^= 1
        else:
            pay = pay[:-1]
            blocks[3] = blocks[3][:hs + len(pay)].copy()
            blocks[3][44:48] = np.frombuffer(np.int32(len(pay)).tobytes(), np.uint8)
        _refit(blocks[3], hs, pay, crc)
        assert lz4_ref.stored_checksums_ok(blocks[3], crc)
        with pytest.raises(zlib.error):
            zlib.decompress(pay.tobytes())
        sizes = np.array([len(x) for x in blocks], dtype=np.int64)
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        with pytest.raises(ob.ObGpuError) as e:
            ob.PageBatch(ctx, type(st)(np.concatenate(blocks), offs, sizes, st.total_rows, st.n_cols), compressor=ZLIB)
        assert e.value.code == ob.OB_INVALID_DATA and "zlib" in ctx.last_error(), what
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=ZLIB)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_string_pointers_address_the_device_image():
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, ZLIB)
    ctx = ob.ScanContext(0)
    cb = ob.PageBatch(ctx, st, compressor=ZLIB)
    base, size = cb.device_image()
    assert base != 0 and size >= table.sizes.sum()
    r = cb.scan(ob.White(1, ob.WHITE_OP_LT, [10]), [3], string_base=base)
    ptrs, lens, _ = r.fetch_col(0)
    h, o = r.fetch_strings(0)

    class DeviceBytes:
        __cuda_array_interface__ = {"shape": (size,), "typestr": "|u1", "data": (base, False), "version": 3}
    dev = torch.as_tensor(DeviceBytes(), device="cuda").cpu().numpy()
    ptrs = ptrs.astype(np.uint64)
    rows = np.arange(len(ptrs))
    for k in rows[:: max(len(rows) // 500, 1)]:
        rel = int(ptrs[k]) - base
        assert 0 <= rel and rel + int(lens[k]) <= size
        assert dev[rel:rel + int(lens[k])].tobytes() == h[o[k]:o[k + 1]].tobytes()
    r.free()
    cb.close()
    ctx.close()


def test_device_compress_still_refuses_zlib():
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.capi import lib
    table, _ = _table(n=2000)
    ctx = ob.ScanContext(0)
    d_img = torch.from_numpy(table.image).cuda()
    d_off = torch.from_numpy(table.offsets.astype(np.int64)).cuda()
    d_sz = torch.from_numpy(table.sizes.astype(np.uint32).view(np.int32)).cuda()
    used = C.c_int64(0)
    code = lib.obgpu_compress_blocks(ctx._h, C.c_void_p(d_img.data_ptr()), C.c_void_p(d_off.data_ptr()), C.c_void_p(d_sz.data_ptr()),
                                     table.n_blocks, ZLIB, 1, None, 0, None, None, C.byref(used))
    assert code == ob.OB_NOT_SUPPORTED
    ctx.close()
