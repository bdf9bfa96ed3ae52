"""zlib-compressed micro-blocks (compressor 4, zlib_1.0) on the CPU side: the committed zlib vectors are self-consistent and
their census covers every decoder branch; the decoder (zlib_decode.cuh) built for the CPU with one lane under AddressSanitizer
and UBSan returns zlib's bytes for every stream and accepts only malformed streams zlib accepts; the writer's streams decode
with Python's zlib; stored-form tables written with compressor 4 decode to the source blocks; compressor-4 macro blocks parse
and walk in the oracle."""
import ctypes as C
import hashlib
import os
import shutil
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import lz4_ref
import oracle_binding as ora
from test_lz4_blocks import compressible_tables, crc32c, oracle_scan

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_zlib_golden as golden  # noqa: E402

ZLIB = 4


def vectors():
    """(streams [(stream, payload)], malformed [(stream, payload length, zlib accepts, sha256 of its output, refusal, strict)],
    census (streams x features), census names)."""
    z = np.load(os.path.join(HERE, "golden", "zlib_vectors.npz"))
    po, so, bo = z["payload_off"], z["stream_off"], z["bad_off"]
    pay = lambda i: z["payloads"][po[i]:po[i + 1]].tobytes()
    streams = [(z["streams"][so[k]:so[k + 1]].tobytes(), pay(i)) for k, i in enumerate(z["stream_payload"])]
    ref, strict = [str(s) for s in z["refusal_names"]], [str(s) for s in z["strict_names"]]
    bad = [(z["bad"][bo[k]:bo[k + 1]].tobytes(), len(pay(i)), bool(z["bad_zlib_ok"][k]), z["bad_zlib_sha256"][k].tobytes(),
            ref[int(z["bad_refusal"][k])], strict[int(z["bad_strict"][k])]) for k, i in enumerate(z["bad_payload"])]
    return streams, bad, z["census"], [str(s) for s in z["census_names"]]


def test_vectors_are_self_consistent_and_cover_every_branch():
    streams, bad, census, names = vectors()
    assert len(streams) >= 150 and len(bad) >= 500 and census.shape == (len(streams), len(names))
    assert names == golden.CENSUS
    for k, (s, p) in enumerate(streams):
        if len(p) <= 20_000:   # the Python walker is slow: the small streams re-check the recorded census
            out, feats = golden.walk(s)
            assert out == p and {names[j] for j in np.nonzero(census[k])[0]} == feats - {"trailing"}, k
    missing = [n for j, n in enumerate(names) if not census[:, j].any()]
    assert not missing, missing
    assert {r for *_, r, _ in bad} == set(golden.REFUSALS)
    assert {s for *_, s in bad} == set(golden.STRICT)
    for s, n, ok, _, r, strict in bad:   # every hand-made stream is refused by zlib, except the one the decoder is stricter on
        if r:
            assert ok == (r == "trailing_bytes"), r
        assert (strict == "trailing_bytes") == (r == "trailing_bytes")
    z = golden.libz()
    if z is None:
        pytest.skip("libz.so.1 not present: verdicts not re-checked")
    for s, p in streams:
        assert golden.uncompress(z, s, len(p)) == p
    for s, n, ok, digest, _, _ in bad:
        out = golden.uncompress(z, s, n)
        assert (out is not None) == ok
        if ok:
            assert hashlib.sha256(out).digest() == digest


@pytest.fixture(scope="module")
def cpu_decoder(tmp_path_factory):
    """tests/cpp/zlib_decode_cpu.cpp (the device decoder's code, one lane) built with AddressSanitizer and UBSan."""
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ not present")
    exe = str(tmp_path_factory.mktemp("zlibd") / "zlib_decode_cpu")
    cmd = [cxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-fsanitize=address,undefined",
           "-fno-sanitize-recover=all", "-o", exe, os.path.join(HERE, "cpp", "zlib_decode_cpu.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(items):
        """items [(stream, n_out)] -> [output bytes or None]"""
        data = b"".join(struct.pack("<qq", len(s), n) + s for s, n in items)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        p = subprocess.run([exe], input=data, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode()[-3000:]
        o, k, outs = p.stdout, 0, []
        for _, n in items:
            st = struct.unpack_from("<i", o, k)[0]
            k += 4
            outs.append(o[k:k + n] if st == 0 else None)
            k += n if st == 0 else 0
        assert k == len(o)
        return outs
    return run


def test_cpu_decoder_returns_zlibs_bytes_and_refuses_what_zlib_refuses(cpu_decoder):
    streams, bad, _, _ = vectors()
    for (s, p), o in zip(streams, cpu_decoder([(s, len(p)) for s, p in streams])):
        assert o == p
    outs = cpu_decoder([(s, n) for s, n, *_ in bad])
    refused_by_zlib_only = set()
    for k, ((s, n, ok, digest, refusal, strict), o) in enumerate(zip(bad, outs)):
        if o is not None:   # accepted: zlib accepts it too, with the same bytes
            assert ok, (k, refusal)
            assert hashlib.sha256(o).digest() == digest, k
        elif ok:            # stricter than zlib only where the vectors say so
            assert strict, (k, refusal)
            refused_by_zlib_only.add(strict)
    assert refused_by_zlib_only == {"trailing_bytes"}


def writer_payloads():
    rng = np.random.default_rng(12)
    rnd = lambda n: rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    head = rnd(300)
    out = {"empty": b"", "one": b"x", "two": b"xy", "three": b"xyz", "twelve": b"abcabcabcabc", "thirteen": b"abcabcabcabca",
           "noise": rnd(100_000), "small_ints": rng.integers(0, 4, size=200_000, dtype=np.uint8).tobytes()}
    for d in (32768, 32769):   # the second copy of `head` lies exactly d bytes back
        out["offset_%d" % d] = head + rnd(d - 300) + head + rnd(40)
    for n in (258, 259, 260, 261, 1000):   # one match of n bytes: symbol 285 at 258, pieces of 3..258 past it
        y = rnd(n)
        out["length_%d" % n] = rnd(20) + y + y + rnd(20)
    out["text"] = b" ".join(rng.choice([b"micro", b"block", b"zlib", b"the"], size=30_000))
    return out


def test_writer_streams_decode_with_python_zlib():
    from oceanbase_b200.sstable import zlib_compress
    streams, _, _, _ = vectors()
    pays = dict(writer_payloads())
    for k, p in enumerate(sorted({p for _, p in streams}, key=len)):
        pays["golden_%d" % k] = p
    for name, p in pays.items():
        z = zlib_compress(p).tobytes()
        assert len(z) <= len(p) + 5 * (len(p) // 32768 + 1) + 7, name
        assert z[:2] == b"\x78\x01", name
        assert zlib.decompress(z) == p, name
        if len(p) > 40_000:   # the Python walker is slow: the features are checked on the shorter payloads
            continue
        out, feats = golden.walk(z)
        assert out == p and "trailing" not in feats, name
        assert feats <= {"stored", "stored_empty", "fixed", "multi_block", "literal", "match", "match_overlap", "len_258",
                         "dist_32768"}, (name, feats)
        if name == "offset_32768":
            assert "dist_32768" in feats
        if name == "noise":
            assert "stored" in feats and len(z) < len(p) + 50
        if name == "length_258":
            assert "len_258" in feats
    assert zlib_compress(b"").tobytes() == b"\x78\x01\x03\x00\x00\x00\x00\x01"


def test_compress_table_zlib_decodes_to_the_source_blocks():
    from oceanbase_b200.sstable import TableImage, compress_table
    for name, table, proj in compressible_tables():
        st = compress_table(table, ZLIB)
        hdr = [lz4_ref.header_fields(st.block(i)) for i in range(st.n_blocks)]
        n_comp = sum(1 for _, ln, zl in hdr if zl < ln)
        assert n_comp >= 0.9 * st.n_blocks, (name, n_comp, st.n_blocks)
        dec = []
        for i in range(st.n_blocks):
            blk = st.block(i)
            assert lz4_ref.stored_checksums_ok(blk, crc32c), (name, i)
            hs, ln, zl = hdr[i]
            src = table.block(i)
            d = blk.copy() if zl == ln else np.concatenate([blk[:hs], np.frombuffer(zlib.decompress(blk[hs:].tobytes()), np.uint8)])
            assert len(d) == hs + ln
            # the decoded copy keeps the stored header: only header_checksum_, data_zlength_ and data_checksum_ differ
            assert np.array_equal(d[64:], src[64:]) and np.array_equal(d[:8], src[:8]) and np.array_equal(d[10:44], src[10:44]), (name, i)
            assert np.array_equal(d[56:64], src[56:64]), (name, i)
            dec.append(d)
        offs = np.concatenate([[0], np.cumsum([len(d) for d in dec])[:-1]]).astype(np.int64)
        decoded = TableImage(np.concatenate(dec), offs, np.array([len(d) for d in dec], dtype=np.int64), table.total_rows, table.n_cols)
        w1, w2 = oracle_scan(table, proj), oracle_scan(decoded, proj)
        assert w1["selected"] == w2["selected"] > 0 and np.array_equal(w1["row_ids"], w2["row_ids"])
        assert np.array_equal(w1["sel_offset"], w2["sel_offset"])
        for c in range(len(proj)):
            if w1["lens"][c] is not None:
                assert np.array_equal(w1["lens"][c], w2["lens"][c])
            else:
                assert np.array_equal(w1["data"][c], w2["data"][c])
            assert np.array_equal(w1["nulls"][c], w2["nulls"][c])


def test_zlib_macro_blocks_parse_and_walk_in_the_oracle():
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    _, table, _ = compressible_tables()[0]
    types = [capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_INT, capi.OBJ_VARCHAR, capi.OBJ_VARCHAR]
    ms = 64 << 10
    mi = build_macro_blocks(table, types, 1, macro_block_size=ms, compressor=capi.COMPRESSOR_ZLIB)
    stored = compress_table(table, ZLIB)
    O = ora.oracle()
    O.ora_macro_block_micro_blocks.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32]
    O.ora_macro_block_parse.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
    k = 0
    for m in range(mi.n_macro):
        blk = np.ascontiguousarray(mi.image[m * ms:(m + 1) * ms])
        f = np.zeros(28, dtype=np.int64)
        assert O.ora_macro_block_parse(blk.ctypes.data, blk.size, f.ctypes.data, 1) == 0
        assert f[25] == ZLIB
        offs, szs, cnt = np.zeros(4096, dtype=np.int64), np.zeros(4096, dtype=np.int64), C.c_int32(0)
        assert O.ora_macro_block_micro_blocks(blk.ctypes.data, blk.size, offs.ctypes.data, szs.ctypes.data, 4096, C.byref(cnt), 1) == 0
        for j in range(cnt.value):
            assert np.array_equal(blk[offs[j]:offs[j] + szs[j]], stored.block(k))
            k += 1
    assert k == table.n_blocks


def test_writer_refuses_compressed_blocks_with_zlib():
    from oceanbase_b200 import capi
    from oceanbase_b200.capi import lib
    from oceanbase_b200.sstable import compress_table
    _, table, _ = compressible_tables()[1]
    st = compress_table(table, ZLIB)
    off, sz = st.offsets.copy(), st.sizes.copy()
    o = np.zeros(st.image.size * 2, dtype=np.uint8)
    oo, osz, used = np.zeros(st.n_blocks, np.int64), np.zeros(st.n_blocks, np.int64), C.c_int64(0)
    assert lib.obgpu_writer_compress_blocks(st.image.ctypes.data, off.ctypes.data, sz.ctypes.data, st.n_blocks, ZLIB, 1,
                                            o.ctypes.data, o.size, oo.ctypes.data, osz.ctypes.data, C.byref(used)) == capi.OB_INVALID_DATA
