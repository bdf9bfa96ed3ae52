"""zstd-compressed micro-blocks (compressor 6) decoded on the device: obgpu_zstd_decompress on every committed libzstd frame and
on the malformed streams (the device's verdict is libzstd's, or stricter only in the cases the vectors name); page batches
opened from compressor-6 blocks made by the writer and by libzstd, and from compressor-6 macro blocks, scan bit for bit like
the plain batch; mixed LZ4 / zstd macro images are refused; corrupt input is refused with OBGPU_INVALID_DATA and the ctx
keeps working; string pointers rebased on obgpu_batch_device_image address the right device bytes."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_gpu_lz4_blocks import _reframe_with, _table, scans_equal
from test_zstd_blocks import vectors, zstd

pytestmark = pytest.mark.gpu
ZSTD = 6


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
    code = lib.obgpu_zstd_decompress(ctx._h, C.c_void_p(d_in.data_ptr()), in_off.ctypes.data, in_len.ctypes.data,
                                     C.c_void_p(d_out.data_ptr()), out_off.ctypes.data, out_len.ctypes.data, len(streams), status.ctypes.data)
    out = d_out.cpu().numpy()
    return code, status, [out[o:o + n].tobytes() for o, n in zip(out_off, out_len)]


def test_zstd_decompress_golden_frames_and_malformed_streams():
    import oceanbase_b200 as ob
    frames, bad, _, _ = vectors()
    ctx = ob.ScanContext(0)
    code, status, outs = _decompress(ctx, [f for f, _ in frames], [len(p) for _, p in frames])
    assert code == 0 and (status == 0).all(), np.nonzero(status)[0]
    for (_, p), o in zip(frames, outs):
        assert o == p
    code, status, outs = _decompress(ctx, [s for s, *_ in bad], [n for _, n, *_ in bad])
    assert code == ob.OB_INVALID_DATA
    stricter = set()
    for k, ((s, n, lib_ok, digest, strict), st, o) in enumerate(zip(bad, status, outs)):
        if st == 0:   # the device accepts only what libzstd accepts, with libzstd's bytes
            assert lib_ok, k
            assert hashlib.sha256(o).digest() == digest, k
        elif lib_ok:  # stricter than libzstd only where RFC 8878 asks for a refusal libzstd does not make
            assert strict, k
            stricter.add(strict)
    assert {"trailing_frame", "skippable_frame", "modes_reserved"} <= stricter
    # the ctx keeps working: the golden frames decode again
    code, status, _ = _decompress(ctx, [f for f, _ in frames[:20]], [len(p) for _, p in frames[:20]])
    assert code == 0 and (status == 0).all()
    ctx.close()


def _libzstd_compress(level, checksum):
    zs = zstd()
    if zs is None:
        pytest.skip("libzstd.so.1 not present")
    return lambda p: zs.compress(p, level, checksum=checksum)


@pytest.mark.parametrize("cs", [False, True])
@pytest.mark.parametrize("source,on_device", [("writer", False), ("writer", True), ("l1", False), ("l3ck", True), ("l19", False)])
def test_zstd_batch_scans_like_the_plain_batch(cs, source, on_device):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(cs=cs, n=20_000 if source != "writer" else 60_000)
    if source == "writer":
        st = compress_table(table, ZSTD)
    else:
        st = _reframe_with(table, _libzstd_compress(int(source[1:3].rstrip("c")), 1 if source.endswith("ck") else 0))
    n_comp = sum(1 for i in range(st.n_blocks) if lz4_ref.header_fields(st.block(i))[2] < lz4_ref.header_fields(st.block(i))[1])
    assert n_comp >= 0.9 * st.n_blocks
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    keep = None
    if on_device:
        keep = torch.from_numpy(st.image).cuda()
        cb = ob.PageBatch(ctx, st, device_image_ptr=keep.data_ptr(), image_size=st.image.size, compressor=ZSTD)
    else:
        cb = ob.PageBatch(ctx, st, compressor=ZSTD)
    assert cb.n_blocks == table.n_blocks and cb.total_rows == table.total_rows
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_mixed_blocks_edge_sizes_and_a_multi_block_frame():
    """Raw and compressed blocks in one batch, a 1-row block and a block above 128 KiB (its frame spans several zstd blocks)."""
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
    big, _ = _table(n=20_000, rpb=20_000)
    assert big.sizes.max() > 128 << 10
    table = TableImage.concat([t1, noise, one, big])
    st = compress_table(table, ZSTD)
    # zstd shrinks even the noise blocks a little: every third block is put back in its plain (raw stored) form
    blocks = [table.block(i) if i % 3 == 1 else st.block(i) for i in range(st.n_blocks)]
    offs = np.concatenate([[0], np.cumsum([len(x) for x in blocks])[:-1]]).astype(np.int64)
    st = TableImage(np.concatenate(blocks), offs, np.array([len(x) for x in blocks], dtype=np.int64), table.total_rows, table.n_cols)
    kinds = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
    assert any(z == l for _, l, z in kinds) and any(z < l for _, l, z in kinds)
    ctx = ob.ScanContext(0)
    plain = ob.PageBatch(ctx, table)
    cb = ob.PageBatch(ctx, st, compressor=ZSTD)
    scans_equal(plain, cb)
    cb.close()
    with pytest.raises(ob.ObGpuError) as e:   # an LZ4 open of zstd payloads fails on the stream, not on the checksum
        ob.PageBatch(ctx, st, compressor=capi.COMPRESSOR_LZ4)
    assert e.value.code == ob.OB_INVALID_DATA
    plain.close()
    ctx.close()


def test_twenty_thousand_block_batch():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=20_000 * 40, rpb=40, seed=4)
    assert table.n_blocks >= 20_000
    st = compress_table(table, ZSTD)
    ctx = ob.ScanContext(0)
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=ZSTD)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


@pytest.mark.parametrize("macro_size,on_device", [(2 << 20, False), (256 << 10, True), (64 << 10, False)])
def test_zstd_macro_blocks_scan_like_the_plain_image(macro_size, on_device):
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import build_macro_blocks
    for cs in (False, True):
        table, types = _table(cs=cs)
        mi = build_macro_blocks(table, types, 1, macro_block_size=macro_size, compressor=ZSTD)
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


def test_macro_image_mixing_lz4_and_zstd_is_refused():
    import oceanbase_b200 as ob
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks
    ms = 64 << 10
    table, types = _table(n=9000)
    a = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=capi.COMPRESSOR_LZ4)
    b = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=ZSTD)
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


def test_corrupt_input_is_refused_and_the_ctx_keeps_working():
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, ZSTD)
    crc = lambda a: int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))
    hs, ln, zl = lz4_ref.header_fields(st.block(3))
    assert zl < ln
    ctx = ob.ScanContext(0)
    # a flipped payload byte: the payload checksum refuses it
    bad = st.image.copy()
    bad[st.offsets[3] + hs + zl // 2] ^= 0x20
    assert not lz4_ref.stored_checksums_ok(bad[st.offsets[3]:st.offsets[3] + st.sizes[3]], crc)
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, type(st)(bad, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=ZSTD)
    assert e.value.code == ob.OB_INVALID_DATA and "checksum" in ctx.last_error()
    # a malformed frame under a correct checksum: Frame_Content_Size one more than data_length_ (the decoder refuses it)
    bad = st.image.copy()
    b = bad[st.offsets[3]:st.offsets[3] + st.sizes[3]]
    pay = b[hs:]
    fhd = int(pay[4])
    assert fhd & 0x20 and (fhd >> 6) == 1            # Single_Segment, 2-byte Frame_Content_Size
    v = int(pay[5]) | (int(pay[6]) << 8)
    pay[5], pay[6] = (v + 1) & 0xff, (v + 1) >> 8
    b[48:56] = np.frombuffer(np.uint64(crc(np.ascontiguousarray(pay))).tobytes(), np.uint8)
    b[8:10] = 0
    b[8:10] = np.frombuffer(np.uint16(lz4_ref.header_checksum_fold(b)).tobytes(), np.uint8)
    assert lz4_ref.stored_checksums_ok(b, crc)
    zs = zstd()
    if zs is not None:
        assert zs.decompress(pay.tobytes(), ln) is None
    with pytest.raises(ob.ObGpuError) as e:
        ob.PageBatch(ctx, type(st)(bad, st.offsets, st.sizes, st.total_rows, st.n_cols), compressor=ZSTD)
    assert e.value.code == ob.OB_INVALID_DATA and "zstd" in ctx.last_error()
    plain, cb = ob.PageBatch(ctx, table), ob.PageBatch(ctx, st, compressor=ZSTD)
    scans_equal(plain, cb)
    cb.close()
    plain.close()
    ctx.close()


def test_string_pointers_address_the_device_image():
    import torch
    import oceanbase_b200 as ob
    from oceanbase_b200.sstable import compress_table
    table, _ = _table(n=9000)
    st = compress_table(table, ZSTD)
    ctx = ob.ScanContext(0)
    cb = ob.PageBatch(ctx, st, compressor=ZSTD)
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
