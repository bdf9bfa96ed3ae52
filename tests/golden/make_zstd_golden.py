"""Writes tests/golden/zstd_vectors.npz: zstd frames (RFC 8878) produced by the system libzstd (libzstd.so.1, loaded with ctypes;
1.5.5 when the vectors were made), malformed streams with libzstd's verdict, and a feature census of every frame.

  frames    : every payload at levels -5, 1, 3, 9 and 19 (large payloads at fewer levels), with Frame_Content_Size and without
              a checksum, plus selected ones with ZSTD_c_checksumFlag=1 and with ZSTD_c_contentSizeFlag=0 (a Window_Descriptor
              and no Frame_Content_Size); "reheader" frames re-encode a libzstd frame's header by hand: Frame_Content_Size in
              8 / 4 / 2 bytes, a Dictionary_ID field holding 0, no Single_Segment.
  malformed : truncations, one-bit flips at spread positions, hand-made bad headers (dictionary ID, reserved bit, reserved
              block type, skippable frame, wrong content size, bad checksum) and two concatenated frames, each with libzstd's
              verdict (ZSTD_decompressDCtx into a buffer of exactly the payload's size must return that size) and, where it
              accepts, the SHA-256 of its output. `strict` names the cases where RFC 8878 asks for a refusal that libzstd 1.5.5 does not make:
              "trailing_frame" (bytes after the first frame), "skippable_frame" (libzstd skips one), "modes_reserved" (a
              flip of the reserved low bits of Symbol_Compression_Modes, which libzstd ignores) and "huffman_stream_end" (a
              flip inside Huffman-coded literal streams: libzstd's fast 4-stream decoder checks the decoded length of each
              stream but not that the stream ends at its first bit).
  census    : a header-only walker records, per frame, the features of census_names (block types, literals types, stream
              counts, Huffman weight encodings, FCS field sizes, checksum flag, Window_Descriptor, LL / OF / ML modes).

  python tests/golden/make_zstd_golden.py
"""
import ctypes as C
import hashlib
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LEVELS = [-5, 1, 3, 9, 19]
CENSUS = ["fcs0", "fcs1", "fcs2", "fcs4", "fcs8", "single_segment", "window_descriptor", "checksum", "block_raw", "block_rle",
          "block_compressed", "multi_block", "lit_raw", "lit_rle", "lit_huffman", "lit_treeless", "streams1", "streams4",
          "weights_direct", "weights_fse", "no_sequences", "ll_predefined", "ll_rle", "ll_fse", "ll_repeat", "of_predefined",
          "of_rle", "of_fse", "of_repeat", "ml_predefined", "ml_rle", "ml_fse", "ml_repeat"]
STRICT = ["", "trailing_frame", "modes_reserved", "huffman_stream_end", "skippable_frame"]


def libzstd():
    try:
        z = C.CDLL("libzstd.so.1")
    except OSError:
        return None
    z.ZSTD_createCCtx.restype = C.c_void_p
    z.ZSTD_createDCtx.restype = C.c_void_p
    z.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    z.ZSTD_CCtx_setParameter.restype = C.c_size_t
    z.ZSTD_CCtx_reset.argtypes = [C.c_void_p, C.c_int]
    z.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]
    z.ZSTD_compress2.restype = C.c_size_t
    z.ZSTD_decompressDCtx.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]
    z.ZSTD_decompressDCtx.restype = C.c_size_t
    z.ZSTD_isError.argtypes = [C.c_size_t]
    z.ZSTD_compressBound.argtypes = [C.c_size_t]
    z.ZSTD_compressBound.restype = C.c_size_t
    z.ZSTD_versionString.restype = C.c_char_p
    return z


class Zstd:
    """libzstd through ctypes: compress(payload, level, checksum, content_size) and decompress(frame, n) -> bytes or None."""

    def __init__(self, z):
        self.z, self.c, self.d = z, z.ZSTD_createCCtx(), z.ZSTD_createDCtx()

    def compress(self, p, level, checksum=0, content_size=1):
        z = self.z
        z.ZSTD_CCtx_reset(self.c, 1)   # ZSTD_reset_session_only
        z.ZSTD_CCtx_setParameter(self.c, 100, level)          # ZSTD_c_compressionLevel
        z.ZSTD_CCtx_setParameter(self.c, 201, checksum)       # ZSTD_c_checksumFlag
        z.ZSTD_CCtx_setParameter(self.c, 200, content_size)   # ZSTD_c_contentSizeFlag
        cap = z.ZSTD_compressBound(len(p))
        buf = C.create_string_buffer(cap)
        n = z.ZSTD_compress2(self.c, buf, cap, bytes(p), len(p))
        assert not z.ZSTD_isError(n)
        return buf.raw[:n]

    def decompress(self, frame, n):
        """ZSTD_decompressDCtx into exactly n bytes: the bytes, or None when libzstd refuses or produces another size."""
        buf = C.create_string_buffer(max(n, 1))
        r = self.z.ZSTD_decompressDCtx(self.d, buf, n, bytes(frame), len(frame))
        return None if self.z.ZSTD_isError(r) or r != n else buf.raw[:n]


def walk(frame):
    """Header-only walk of one frame: (set of CENSUS features, byte offsets of Symbol_Compression_Modes bytes, [start, end)
    byte ranges of Huffman-coded literal streams)."""
    f, modes_at, huf = set(), [], []
    fhd = frame[4]
    fcs_flag, single, did = fhd >> 6, (fhd >> 5) & 1, fhd & 3
    f.add("single_segment" if single else "window_descriptor")
    if (fhd >> 2) & 1:
        f.add("checksum")
    fcs = [1 if single else 0, 2, 4, 8][fcs_flag]
    f.add("fcs%d" % fcs)
    p = 5 + (0 if single else 1) + [0, 1, 2, 4][did] + fcs
    nblocks = 0
    while True:
        bh = int.from_bytes(frame[p:p + 3], "little")
        p += 3
        bt, bs = (bh >> 1) & 3, bh >> 3
        nblocks += 1
        f.add(["block_raw", "block_rle", "block_compressed"][bt])
        if bt == 2:
            b = frame[p:p + bs]
            lt, sf = b[0] & 3, (b[0] >> 2) & 3
            if lt <= 1:
                lh = [1, 2, 1, 3][sf]
                size = b[0] >> 3 if lh == 1 else int.from_bytes(b[:lh], "little") >> 4
                q = lh + (size if lt == 0 else 1)
                f.add("lit_raw" if lt == 0 else "lit_rle")
            else:
                lh = [3, 3, 4, 5][sf]
                v = int.from_bytes(b[:lh], "little")
                csize = [(v >> 14) & 0x3ff, (v >> 14) & 0x3ff, v >> 18, v >> 22][sf]
                f.add("streams1" if sf == 0 else "streams4")
                f.add("lit_huffman" if lt == 2 else "lit_treeless")
                tree = 0
                if lt == 2:
                    f.add("weights_direct" if b[lh] >= 128 else "weights_fse")
                    tree = 1 + ((b[lh] - 127 + 1) // 2 if b[lh] >= 128 else b[lh])
                huf.append((p + lh + tree, p + lh + csize))
                q = lh + csize
            ns = b[q]
            q += 1 if ns < 128 else 2 if ns < 255 else 3
            if ns == 0:
                f.add("no_sequences")
            else:
                m = b[q]
                modes_at.append(p + q)
                for name, mode in (("ll", m >> 6), ("of", (m >> 4) & 3), ("ml", (m >> 2) & 3)):
                    f.add(name + "_" + ["predefined", "rle", "fse", "repeat"][mode])
            p += bs
        else:
            p += 1 if bt == 1 else bs
        if bh & 1:
            break
    if nblocks > 1:
        f.add("multi_block")
    return f, modes_at, huf


def reheader(frame, fcs_bytes=None, dict_id0=False, no_single=False):
    """The same blocks under a hand-encoded frame header: Frame_Content_Size in fcs_bytes bytes (8, 4 or 2), a Dictionary_ID
    field of 0, or no Single_Segment (a Window_Descriptor covering the content)."""
    fhd = frame[4]
    single, did = (fhd >> 5) & 1, fhd & 3
    fcs_len = [1 if single else 0, 2, 4, 8][fhd >> 6]
    hdr_end = 5 + (0 if single else 1) + [0, 1, 2, 4][did] + fcs_len
    raw = frame[hdr_end - fcs_len:hdr_end]
    fcs = int.from_bytes(raw, "little") + (256 if fcs_len == 2 else 0)
    nb = fcs_bytes or (8 if fcs >= 1 << 32 else 4 if fcs >= 65536 + 256 else 2 if fcs >= 256 else 1)
    flag = {1: 0, 2: 1, 4: 2, 8: 3}[nb]
    out = bytearray(frame[:4])
    out.append((flag << 6) | ((0 if no_single else 1) << 5) | (fhd & 4) | (1 if dict_id0 else 0))
    if no_single:
        wl = max(10, (max(fcs, 1) - 1).bit_length())
        out.append((wl - 10) << 3)
    if dict_id0:
        out.append(0)
    if not (no_single and nb == 1):   # without Single_Segment, FCS flag 0 means no field
        out += (fcs - (256 if nb == 2 else 0)).to_bytes(nb, "little")
    return bytes(out) + frame[hdr_end:]


def payloads():
    rng = np.random.default_rng(20261015)
    rnd = lambda n: rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    words = [b"micro", b"block", b"header", b"column", b"scan", b"offset", b"the", b"of", b"zstd", b"sstable"]
    text = lambda n: b" ".join(words[i] for i in rng.integers(0, len(words), size=n))
    out = [(b"", "all"), (b"a", "all"), (rnd(7), "all"), (rnd(200), "all"), (bytes(255), "all"), (bytes(256), "all"),
           (rnd(1000), "all"),
           (rng.integers(0, 16, size=3000, dtype=np.uint8).tobytes(), "all"),                        # direct Huffman weights
           (text(800), "all"), (text(1500), "all"),
           (np.cumsum(rng.integers(0, 100, size=1000)).astype(np.int64).tobytes(), "all"),
           (rng.integers(0, 40, size=2000).astype(np.int64).tobytes(), "all"),
           (bytes(300_000), "few"),                                                                  # RLE blocks
           (text(25_000), "9+19")]                                                                   # 145 KB text: OF / ML repeat
    # a pool of 40-byte random chunks padded with zeros to the first 128 KiB block, then permutations of the pool, each chunk
    # followed by one constant byte: from the second block on, level 19 codes only matches of one length and literals of one
    # value (RLE literals, ML RLE mode, repeated LL / ML tables)
    prng = np.random.default_rng(3)
    pool = [prng.integers(0, 256, size=40, dtype=np.uint8).tobytes() for _ in range(400)]
    head = b"".join(pool)
    out.append((head + bytes((128 << 10) - len(head)) +
                b"".join(b"".join(pool[i] + b"\x07" for i in prng.permutation(len(pool))) for _ in range(12)), "19"))
    for d in (1, 3, 17, 1000):                                                                      # repeats at distance d
        pat = rnd(d)
        out.append((rnd(20) + pat * (2 + 3000 // d) + rnd(20), "all"))
    return out


def main():
    z = libzstd()
    assert z is not None, "libzstd.so.1 is required to make the vectors"
    zs = Zstd(z)
    pays = payloads()
    frames, f_pay, f_kind, kinds = [], [], [], ["level", "checksum", "no_content_size", "reheader"]
    for i, (p, which) in enumerate(pays):
        levels = LEVELS if which == "all" else [1, 19] if which == "few" else [int(v) for v in which.split("+")]
        for lv in levels:
            frames.append((zs.compress(p, lv), i, 0))
        if which in ("all", "few"):
            frames.append((zs.compress(p, 3, checksum=1), i, 1))
            frames.append((zs.compress(p, 19 if which == "few" else 9, checksum=1, content_size=0), i, 2))
        if which == "all" and len(p) > 0:
            base = zs.compress(p, 3)
            for kw in ({"fcs_bytes": 8}, {"fcs_bytes": 4}, {"dict_id0": True}, {"no_single": True}):
                frames.append((reheader(base, **kw), i, 3))
            if 256 <= len(p) < 65536 + 256:
                frames.append((reheader(base, fcs_bytes=2), i, 3))
    for fr, i, _ in frames:
        assert zs.decompress(fr, len(pays[i][0])) == pays[i][0], i
    census = np.zeros((len(frames), len(CENSUS)), dtype=np.uint8)
    for k, (fr, _, _) in enumerate(frames):
        feats, _, _ = walk(fr)
        for name in feats:
            census[k, CENSUS.index(name)] = 1
    # malformed streams: (stream, payload index, strict reason)
    bad = []
    rng = np.random.default_rng(7)
    for k, (fr, i, kind) in enumerate(frames):
        if kind != 0 or len(fr) > 4_000:
            continue
        _, modes_at, huf = walk(fr)
        for cut in sorted({len(fr) - 1, len(fr) // 2, 6}):
            if cut < len(fr):
                bad.append((fr[:cut], i, 0))
        for at in sorted(set(rng.integers(4, len(fr), size=min(8, len(fr) - 4)).tolist()) | set(modes_at[:1])):
            t = bytearray(fr)
            bit = 1 << int(rng.integers(0, 8)) if at not in modes_at else 1 << int(rng.integers(0, 2))
            t[at] ^= bit
            in_huf = any(a <= at < b for a, b in huf)
            bad.append((bytes(t), i, 2 if at in modes_at else 3 if in_huf else 0))
    p0, fr0 = 9, next(fr for fr, i, kd in frames if i == 9 and kd == 0)          # text payload, level -5
    fhd = fr0[4]
    bad.append((fr0[:4] + bytes([fhd | 1, 7]) + fr0[5:], p0, 0))                     # Dictionary_ID 7
    bad.append((fr0[:4] + bytes([fhd | 8]) + fr0[5:], p0, 0))                        # reserved bit
    hdr_end = 5 + [1, 2, 4, 8][fhd >> 6]
    t = bytearray(fr0)
    t[hdr_end] |= 6                                                                 # reserved block type 3
    bad.append((bytes(t), p0, 0))
    bad.append((b"\x50\x2a\x4d\x18" + (4).to_bytes(4, "little") + b"abcd" + fr0, p0, 4))   # skippable frame first
    fcs_wrong = bytearray(fr0)
    fcs_wrong[5] ^= 1                                                               # Frame_Content_Size off by one
    bad.append((bytes(fcs_wrong), p0, 0))
    ck = next(fr for fr, i, kd in frames if i == p0 and kd == 1)
    bad.append((ck[:-1] + bytes([ck[-1] ^ 0x10]), p0, 0))                          # content checksum
    small = next(fr for fr, i, kd in frames if i == 2 and kd == 0)
    empty = next(fr for fr, i, kd in frames if i == 0 and kd == 0)
    bad.append((small + small, 2, 0))                                               # two frames: 14 bytes for 7
    bad.append((small + empty, 2, 1))                                               # a second, empty frame
    bad.append((small + b"\x00", 2, 0))                                            # one trailing byte
    outs = [zs.decompress(s, len(pays[i][0])) for s, i, _ in bad]
    verdict = np.array([o is not None for o in outs], dtype=np.uint8)
    digest = np.array([np.frombuffer(hashlib.sha256(o).digest() if o is not None else bytes(32), dtype=np.uint8) for o in outs])
    cat = lambda bs: (np.frombuffer(b"".join(bs), dtype=np.uint8),
                      np.concatenate([[0], np.cumsum([len(b) for b in bs])]).astype(np.int64))
    pay, pay_off = cat([p for p, _ in pays])
    fr, fr_off = cat([f for f, _, _ in frames])
    bd, bd_off = cat([s for s, _, _ in bad])
    np.savez_compressed(os.path.join(HERE, "zstd_vectors.npz"), payloads=pay, payload_off=pay_off, frames=fr, frame_off=fr_off,
                        frame_payload=np.array([i for _, i, _ in frames], dtype=np.int32),
                        frame_kind=np.array([kd for _, _, kd in frames], dtype=np.int32), kinds=np.array(kinds),
                        bad=bd, bad_off=bd_off, bad_payload=np.array([i for _, i, _ in bad], dtype=np.int32),
                        bad_strict=np.array([s for _, _, s in bad], dtype=np.int32), strict_names=np.array(STRICT),
                        bad_libzstd_ok=verdict, bad_libzstd_sha256=digest, census=census, census_names=np.array(CENSUS),
                        zstd_version=np.array(z.ZSTD_versionString().decode()))
    miss = [CENSUS[j] for j in range(len(CENSUS)) if not census[:, j].any()]
    print(f"{len(pays)} payloads, {len(frames)} frames, {len(bad)} malformed ({int(verdict.sum())} accepted by libzstd), "
          f"libzstd {z.ZSTD_versionString().decode()}, census misses {miss}")


if __name__ == "__main__":
    main()
