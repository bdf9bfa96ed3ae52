"""Compressed micro-blocks on the CPU side: the LZ4 checker decoder (tests/lz4_ref.py) against liblz4 known answers and
hand-written spec vectors, the writer's LZ4 compressor (decoded by the checker and, when the system liblz4 loads, by
LZ4_decompress_safe), malformed streams refused with liblz4's verdict, and stored-form tables from the writer: mostly
compressed, decoding byte-identical to the source blocks, checksums valid, oracle scans unchanged, macro blocks with
compressor 2 and 7 parsed and walked by the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora

HERE = os.path.dirname(os.path.abspath(__file__))


def liblz4():
    try:
        lz = C.CDLL("liblz4.so.1")
    except OSError:
        return None
    lz.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    return lz


def lz4_safe(lz, stream, out_len):
    """LZ4_decompress_safe into exactly out_len bytes: the decoded bytes, or None when liblz4 refuses the stream or
    produces another size."""
    buf = C.create_string_buffer(max(out_len, 1))
    n = lz.LZ4_decompress_safe(bytes(stream), buf, len(stream), out_len)
    return buf.raw[:n] if n == out_len else None


def vectors():
    z = np.load(os.path.join(HERE, "golden", "lz4_vectors.npz"))
    pay, po, st, so = z["payloads"], z["payload_off"], z["streams"], z["stream_off"]
    out = []
    for k, pi in enumerate(z["payload_index"]):
        out.append((bytes(st[so[k]:so[k + 1]]), bytes(pay[po[pi]:po[pi + 1]]), str(z["kinds"][z["kind"][k]])))
    return out


def crc32c(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return int(ora.oracle().ora_crc64_sse42(0, a.ctypes.data, a.size))


def test_committed_vectors_decode_to_their_payloads():
    vs = vectors()
    assert len(vs) >= 150
    assert {k for _, _, k in vs} == {"default", "fast1", "fast8", "fast64", "hc9"}
    for stream, payload, kind in vs:
        assert lz4_ref.lz4_decompress(stream, len(payload)) == payload, (kind, len(payload))


# hand-written blocks of the format description: (stream, decoded)
SPEC_VECTORS = [
    (bytes([0x50]) + b"hello", b"hello"),                                                        # literals only
    (bytes([0x00]), b""),                                                                        # empty block: one empty token
    (bytes([0x44]) + b"abcd" + bytes([4, 0, 0x50]) + b"efghi", b"abcdabcdabcdefghi"),            # match at distance 4
    (bytes([0x14]) + b"x" + bytes([1, 0, 0x50]) + b"hello", b"x" * 9 + b"hello"),               # overlapping match, distance 1
    (bytes([0xF0, 0x00]) + b"L" * 15, b"L" * 15),                                                # 15 literals: extension byte 0
    (bytes([0x2F]) + b"ab" + bytes([2, 0, 0x03, 0x50]) + b"vwxyz", b"ab" * 12 + b"vwxyz"),      # match length 15 + 3 + 4 = 22
]


def test_hand_written_spec_vectors():
    lz = liblz4()
    for stream, want in SPEC_VECTORS:
        assert lz4_ref.lz4_decompress(stream, len(want)) == want
        if lz is not None and want:
            assert lz4_safe(lz, stream, len(want)) == want


def test_writer_compressor_round_trip():
    from oceanbase_b200.sstable import lz4_compress
    lz = liblz4()
    pays = sorted({p for _, p, _ in vectors()}, key=len)
    rng = np.random.default_rng(5)
    pays += [bytes(rng.integers(0, 4, size=n, dtype=np.uint8)) for n in (13, 17, 100, 4097, 70_000)]
    for p in pays:
        z = lz4_compress(p).tobytes()
        assert len(z) <= len(p) + len(p) // 255 + 16
        assert lz4_ref.lz4_decompress(z, len(p)) == p, len(p)
        if lz is not None:
            assert lz4_safe(lz, z, len(p)) == p, len(p)


def malformed():
    """(name, stream, expected decoded size): each breaks one acceptance rule."""
    good = bytes([0x44]) + b"abcd" + bytes([4, 0, 0x50]) + b"efghi"   # -> 17 bytes
    return [
        ("offset 0", bytes([0x44]) + b"abcd" + bytes([0, 0, 0x50]) + b"efghi", 17),
        ("offset past the produced bytes", bytes([0x44]) + b"abcd" + bytes([5, 0, 0x50]) + b"efghi", 17),
        ("literal run past the input", bytes([0x90]) + b"abcd", 9),
        ("literal extension past the input", bytes([0xF0, 0xFF, 0xFF]), 600),
        ("match extension past the input", bytes([0x4F]) + b"abcd" + bytes([4, 0, 0xFF, 0xFF]), 600),
        ("output shorter than expected", good, 18),
        ("output longer than expected", good, 16),
        ("trailing bytes", good + b"\x00\x00", 17),
        ("empty input", b"", 5),
        ("truncated after the literals", bytes([0x44]) + b"abcd" + bytes([4]), 17),
    ]


def test_malformed_streams_are_refused():
    lz = liblz4()
    for name, stream, n in malformed():
        with pytest.raises(lz4_ref.Lz4Error):
            lz4_ref.lz4_decompress(stream, n)
        # liblz4 reaches the same verdict; it does not test the zero offset the format calls invalid (it copies the
        # bytes in place), so that one stream is the checker's rule alone
        if lz is not None and name != "offset 0":
            assert lz4_safe(lz, stream, n) is None, name


def compressible_tables():
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import Column, encode_table
    rng = np.random.default_rng(11)
    n = 24_000
    key = np.arange(n, dtype=np.int64) * 3 + 1
    small = rng.integers(0, 40, size=n, dtype=np.int64)
    nl = (rng.random(n) < 0.05).astype(np.uint8)
    strs = [b"customer-%04d" % (i % 97) for i in range(n)]
    const = np.full(n, 7, dtype=np.int64)
    hexs = [b"%08x" % (i % 50) for i in range(n)]
    T = capi
    pax = [Column(T.OBJ_INT, T.ENC_RAW, key), Column(T.OBJ_INT, T.ENC_RAW, small, nulls=nl), Column(T.OBJ_VARCHAR, T.ENC_RAW, strs),
           Column(T.OBJ_INT, T.ENC_DICT, small), Column(T.OBJ_INT, T.ENC_CONST, const), Column(T.OBJ_INT, T.ENC_INTEGER_BASE_DIFF, key),
           Column(T.OBJ_VARCHAR, T.ENC_DICT, strs), Column(T.OBJ_VARCHAR, T.ENC_HEX_PACKING, hexs)]
    cs = [Column(T.OBJ_INT, T.ENC_CS_INTEGER, key), Column(T.OBJ_INT, T.ENC_CS_INT_DICT, small, nulls=nl),
          Column(T.OBJ_VARCHAR, T.ENC_CS_STRING, strs), Column(T.OBJ_VARCHAR, T.ENC_CS_STR_DICT, strs)]
    return [("pax", encode_table(pax, 700, rowkey_cnt=1), [0, 1, 2, 3, 4, 5, 6]),
            ("cs", encode_table(cs, 700, rowkey_cnt=1), [0, 1, 2, 3])]


@pytest.mark.parametrize("compressor", [2, 7])
def test_compress_table_decodes_to_the_source_blocks(compressor):
    from oceanbase_b200.sstable import compress_table
    for name, table, proj in compressible_tables():
        st = compress_table(table, compressor)
        hdr = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
        n_comp = sum(1 for _, ln, zl in hdr if zl < ln)
        assert n_comp >= 0.9 * st.n_blocks, (name, n_comp, st.n_blocks)
        dec = []
        for i in range(st.n_blocks):
            blk = st.block(i)
            assert lz4_ref.stored_checksums_ok(blk, crc32c), (name, i)
            d = lz4_ref.micro_block_decompress(blk, compressor)
            src = table.block(i)
            # the decoded copy keeps the stored header: only header_checksum_, data_zlength_ and data_checksum_ differ from
            # the source's; everything behind the header is the source's
            assert np.array_equal(d[64:], src[64:]) and np.array_equal(d[:8], src[:8]) and np.array_equal(d[10:44], src[10:44]), (name, i)
            assert np.array_equal(d[56:64], src[56:64]), (name, i)
            dec.append(d)
        # oracle scans over the decoded blocks equal scans over the originals
        from oceanbase_b200.sstable import TableImage
        offs = np.concatenate([[0], np.cumsum([len(d) for d in dec])[:-1]]).astype(np.int64)
        decoded = TableImage(np.concatenate(dec), offs, np.array([len(d) for d in dec], dtype=np.int64), table.total_rows, table.n_cols)
        w1, w2 = oracle_scan(table, proj), oracle_scan(decoded, proj)
        assert w1["selected"] == w2["selected"] > 0 and np.array_equal(w1["row_ids"], w2["row_ids"])
        assert np.array_equal(w1["sel_offset"], w2["sel_offset"])
        for c in range(len(proj)):
            if w1["lens"][c] is not None:   # string pointers address each image; their lengths must agree
                assert np.array_equal(w1["lens"][c], w2["lens"][c])
            else:
                assert np.array_equal(w1["data"][c], w2["data"][c])
            assert np.array_equal(w1["nulls"][c], w2["nulls"][c])


def oracle_scan(table, proj):
    import oceanbase_b200 as ob
    is_str = [p == 2 or p == 6 for p in proj] if len(proj) > 4 else [p >= 2 for p in proj]
    return ora.scan_table(table, ob.White(1, ob.WHITE_OP_LT, [20]), proj, is_str, [8] * len(proj))


def test_raw_blocks_keep_their_bytes():
    """A block that does not shrink is stored raw, byte for byte; NONE copies every block."""
    from oceanbase_b200.sstable import Column, compress_table, encode_table
    from oceanbase_b200 import capi
    rng = np.random.default_rng(2)
    t = encode_table([Column(capi.OBJ_INT, capi.ENC_RAW, rng.integers(-(1 << 62), 1 << 62, size=3000, dtype=np.int64))], 500)
    for comp in (capi.COMPRESSOR_NONE, capi.COMPRESSOR_LZ4):
        st = compress_table(t, comp)
        assert np.array_equal(st.sizes, t.sizes)
        for i in range(t.n_blocks):
            assert np.array_equal(st.block(i), t.block(i))


@pytest.mark.parametrize("compressor", [2, 7])
def test_compressed_macro_blocks_parse_and_walk_in_the_oracle(compressor):
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    _, table, _ = compressible_tables()[0]
    types = [capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_VARCHAR]
    ms = 64 << 10
    mi = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=compressor)
    stored = compress_table(table, compressor)
    O = ora.oracle()
    O.ora_macro_block_micro_blocks.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32]
    O.ora_macro_block_parse.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    k = 0
    for m in range(mi.n_macro):
        blk = np.ascontiguousarray(mi.image[m * ms:(m + 1) * ms])
        f = np.zeros(28, dtype=np.int64)
        assert O.ora_macro_block_parse(blk.ctypes.data, blk.size, f.ctypes.data, 1) == 0
        assert f[25] == compressor
        offs, szs, cnt = np.zeros(4096, dtype=np.int64), np.zeros(4096, dtype=np.int64), C.c_int32(0)
        assert O.ora_macro_block_micro_blocks(blk.ctypes.data, blk.size, offs.ctypes.data, szs.ctypes.data, 4096, C.byref(cnt), 1) == 0
        for j in range(cnt.value):
            assert np.array_equal(blk[offs[j]:offs[j] + szs[j]], stored.block(k))
            k += 1
    assert k == table.n_blocks
    # the default path writes what it always wrote: compressor_type_ NONE, plain blocks
    plain = build_macro_blocks(table, types, 1, macro_block_size=ms)
    assert plain.image[24 + 104] == capi.COMPRESSOR_NONE


def test_writer_refuses_what_it_cannot_store():
    from oceanbase_b200 import capi
    from oceanbase_b200.capi import lib
    from oceanbase_b200.sstable import compress_table
    _, table, _ = compressible_tables()[1]
    st = compress_table(table, capi.COMPRESSOR_LZ4)
    off, sz = st.offsets.copy(), st.sizes.copy()
    o = np.zeros(st.image.size * 2, dtype=np.uint8)
    oo, osz, used = np.zeros(st.n_blocks, np.int64), np.zeros(st.n_blocks, np.int64), C.c_int64(0)
    # already compressed blocks are not re-framed again; zstd (5) is not written
    assert lib.obgpu_writer_compress_blocks(st.image.ctypes.data, off.ctypes.data, sz.ctypes.data, st.n_blocks, capi.COMPRESSOR_LZ4, 1,
                                            o.ctypes.data, o.size, oo.ctypes.data, osz.ctypes.data, C.byref(used)) == capi.OB_INVALID_DATA
    t_off, t_sz = table.offsets.copy(), table.sizes.copy()
    assert lib.obgpu_writer_compress_blocks(table.image.ctypes.data, t_off.ctypes.data, t_sz.ctypes.data, table.n_blocks, 5, 1,
                                            o.ctypes.data, o.size, oo.ctypes.data, osz.ctypes.data, C.byref(used)) == capi.OB_NOT_SUPPORTED
