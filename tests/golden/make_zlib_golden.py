"""Writes tests/golden/zlib_vectors.npz: zlib streams (RFC 1950 / RFC 1951) made by the system zlib (Python's zlib module for
compression, libz.so.1's uncompress through ctypes for every verdict; 1.3 when the vectors were made), hand-made streams,
malformed streams with zlib's verdict, and a census of the decoder branches each stream reaches.

  streams   : every payload at levels 0, 1, 6 and 9 (default strategy) and at level 6 with Z_FILTERED, Z_HUFFMAN_ONLY (dynamic
              blocks that use no distance), Z_RLE and Z_FIXED; sync / full-flush streams (empty stored blocks); a
              fast_level0_compress-style stream (78 01, stored blocks of <= 65535 bytes, Adler-32); hand-made streams: a
              distance of exactly 32768 and length 258 (symbol 285) in a fixed block, a dynamic block with no distance code
              at all, one with a single distance code of length 1 (the incomplete code inflate accepts), 15-bit codes
              (symbol counts growing 1.7x through Z_HUFFMAN_ONLY), code-length repeats 16 / 17 / 18.
  malformed : truncations, one-bit flips, and one hand-made stream per refusal the decoder makes (bad CM / CINFO / FCHECK,
              FDICT, BTYPE 3, LEN != ~NLEN, HLIT > 286, HDIST > 30, repeat 16 first, a run past HLIT + HDIST, over-subscribed
              and incomplete codes, no end-of-block code, symbols 286 / 287 and 30 / 31, a distance beyond the output, a wrong
              Adler-32, an output longer or shorter than expected), each with zlib's verdict (uncompress into exactly the
              payload's size must return Z_OK with that size) and, where it accepts, the SHA-256 of its output. `strict`
              names the one case where the decoder refuses what uncompress accepts: "trailing_bytes" (bytes after the
              Adler-32, which uncompress ignores).
  census    : `walk` (a plain inflate in Python) records, per stream, the CENSUS features it reaches; `refusal` names the
              REFUSALS branch each hand-made malformed stream is built to reach.

  python tests/golden/make_zlib_golden.py
"""
import ctypes as C
import hashlib
import os
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CENSUS = ["stored", "stored_empty", "fixed", "dynamic", "multi_block", "literal", "match", "match_overlap", "len_258",
          "dist_32768", "code_15bit", "cl_repeat16", "cl_repeat17", "cl_repeat18", "no_dist_code", "single_dist_code",
          "cinfo_lt7", "stored_65535"]
REFUSALS = ["", "header_cm", "header_cinfo", "header_fcheck", "fdict", "btype3", "stored_nlen", "hlit", "hdist", "repeat_first",
            "run_past", "oversubscribed", "incomplete_cl", "incomplete_lit", "incomplete_dist", "missing_eob", "lit_286",
            "dist_30", "dist_too_far", "adler", "output_long", "output_short", "truncated", "trailing_bytes"]
STRICT = ["", "trailing_bytes"]
ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
DL = [5] * 28 + [4, 4]   # a complete code over the 30 distance symbols


def libz():
    try:
        z = C.CDLL("libz.so.1")
    except OSError:
        return None
    z.uncompress.argtypes = [C.c_void_p, C.POINTER(C.c_ulong), C.c_char_p, C.c_ulong]
    z.zlibVersion.restype = C.c_char_p
    return z


def uncompress(z, stream, n):
    """zlib's uncompress into a buffer of exactly n bytes: the bytes, or None unless it returns Z_OK with n bytes."""
    buf = C.create_string_buffer(max(n, 1))
    dl = C.c_ulong(n)
    r = z.uncompress(buf, C.byref(dl), bytes(stream), len(stream))
    return buf.raw[:n] if r == 0 and dl.value == n else None


def compress(p, level, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, strategy)
    return c.compress(p) + c.flush()


# ---- a plain inflate (RFC 1951 as zlib's inflate reads it), for the census ----------------------------------------------
class Bad(Exception):
    pass


class _Bits:
    def __init__(self, b, at):
        self.b, self.pos = b, at * 8

    def take(self, k):
        v = 0
        for j in range(k):
            if self.pos >> 3 >= len(self.b):
                raise Bad("truncated")
            v |= ((self.b[self.pos >> 3] >> (self.pos & 7)) & 1) << j
            self.pos += 1
        return v


def _code(lens, kind):
    """{(length, code): symbol}, or Bad as inflate_table refuses (kind: 'cl', 'lit', 'dist')."""
    count = [0] * 16
    for v in lens:
        count[v] += 1
    mx = max([l for l in range(1, 16) if count[l]], default=0)
    if mx == 0:
        if kind == "cl":
            raise Bad("incomplete_cl")
        return {}
    left = 1
    for l in range(1, 16):
        left = (left << 1) - count[l]
        if left < 0:
            raise Bad("oversubscribed")
    if left > 0 and (kind == "cl" or mx != 1):
        raise Bad("incomplete_" + kind)
    nxt, code = [0] * 16, 0
    count[0] = 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[(l, nxt[l])] = s
            nxt[l] += 1
    return out


def _sym(br, table, feats):
    code = 0
    for l in range(1, 16):
        code = (code << 1) | br.take(1)
        if (l, code) in table:
            if l == 15:
                feats.add("code_15bit")
            return table[(l, code)]
    raise Bad("invalid_code")


def _len_base(c):
    return (3 + c, 0) if c < 8 else (258, 0) if c == 28 else ((((4 + (c & 3)) << ((c >> 2) - 1)) + 3), (c >> 2) - 1)


def _dist_base(d):
    return (d + 1, 0) if d < 4 else ((((2 + (d & 1)) << ((d >> 1) - 1)) + 1), (d >> 1) - 1)


def walk(s):
    """Inflate one zlib stream: (output bytes, set of CENSUS features); raises Bad(reason) where zlib's inflate refuses."""
    f = set()
    if len(s) < 2:
        raise Bad("truncated")
    cmf, flg = s[0], s[1]
    if cmf & 15 != 8:
        raise Bad("header_cm")
    if cmf >> 4 > 7:
        raise Bad("header_cinfo")
    if (cmf * 256 + flg) % 31:
        raise Bad("header_fcheck")
    if flg & 0x20:
        raise Bad("fdict")
    if cmf >> 4 < 7:
        f.add("cinfo_lt7")
    br, out, nblk = _Bits(s, 2), bytearray(), 0
    while True:
        last, bt = br.take(1), br.take(2)
        nblk += 1
        if bt == 0:
            f.add("stored")
            br.pos = (br.pos + 7) & ~7
            at = br.pos >> 3
            if at + 4 > len(s):
                raise Bad("truncated")
            ln, nl = s[at] | s[at + 1] << 8, s[at + 2] | s[at + 3] << 8
            if ln != (~nl & 0xffff):
                raise Bad("stored_nlen")
            if at + 4 + ln > len(s):
                raise Bad("truncated")
            f.add("stored_empty" if ln == 0 else "stored_65535" if ln == 65535 else "stored")
            out += s[at + 4:at + 4 + ln]
            br.pos = (at + 4 + ln) * 8
        elif bt == 3:
            raise Bad("btype3")
        else:
            if bt == 1:
                f.add("fixed")
                lit = _code([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, "lit")
                dist = _code([5] * 32, "dist")
            else:
                f.add("dynamic")
                nlen, ndist, ncode = br.take(5) + 257, br.take(5) + 1, br.take(4) + 4
                if nlen > 286:
                    raise Bad("hlit")
                if ndist > 30:
                    raise Bad("hdist")
                cl = [0] * 19
                for k in range(ncode):
                    cl[ORDER[k]] = br.take(3)
                clt = _code(cl, "cl")
                lens = []
                while len(lens) < nlen + ndist:
                    sym = _sym(br, clt, set())
                    if sym < 16:
                        lens.append(sym)
                        continue
                    if sym == 16:
                        if not lens:
                            raise Bad("repeat_first")
                        v, r = lens[-1], 3 + br.take(2)
                    else:
                        v, r = 0, 3 + br.take(3) if sym == 17 else 11 + br.take(7)
                    f.add("cl_repeat%d" % sym)
                    if len(lens) + r > nlen + ndist:
                        raise Bad("run_past")
                    lens += [v] * r
                if lens[256] == 0:
                    raise Bad("missing_eob")
                lit = _code(lens[:nlen], "lit")
                dl = lens[nlen:]
                dist = _code(dl, "dist")
                nz = sum(1 for v in dl if v)
                f.add("no_dist_code" if nz == 0 else "single_dist_code" if nz == 1 else "dynamic")
            while True:
                sym = _sym(br, lit, f)
                if sym < 256:
                    f.add("literal")
                    out.append(sym)
                    continue
                if sym == 256:
                    break
                if sym > 285:
                    raise Bad("lit_286")
                base, e = _len_base(sym - 257)
                ln = base + br.take(e)
                ds = _sym(br, dist, f)
                if ds > 29:
                    raise Bad("dist_30")
                base, e = _dist_base(ds)
                d = base + br.take(e)
                if d > len(out):
                    raise Bad("dist_too_far")
                f.add("match")
                if ln == 258:
                    f.add("len_258")
                if d == 32768:
                    f.add("dist_32768")
                if d < ln:
                    f.add("match_overlap")
                for _ in range(ln):
                    out.append(out[-d])
        if last:
            break
    if nblk > 1:
        f.add("multi_block")
    at = (br.pos + 7) >> 3
    if at + 4 > len(s):
        raise Bad("truncated")
    if int.from_bytes(s[at:at + 4], "big") != zlib.adler32(bytes(out)):
        raise Bad("adler")
    if at + 4 != len(s):
        f.add("trailing")
    return bytes(out), f


# ---- hand-made streams ---------------------------------------------------------------------------------------------------
class BitW:
    def __init__(self):
        self.o, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, k):
        self.acc |= v << self.n
        self.n += k
        while self.n >= 8:
            self.o.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, ln):
        self.put(int(format(c, "0%db" % ln)[::-1], 2) if ln else 0, ln)

    def align(self):
        if self.n:
            self.o.append(self.acc & 255)
        self.acc = self.n = 0


def canon(lens):
    count = [0] * 16
    for v in lens:
        count[v] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    codes = {}
    for s, l in enumerate(lens):
        if l:
            codes[s] = (nxt[l], l)
            nxt[l] += 1
    return codes


def len_sym(n):
    if n == 258:
        return 285, 0, 0
    for c in range(27, -1, -1):
        b, e = _len_base(c)
        if b <= n:
            return 257 + c, e, n - b


def dist_sym(d):
    for c in range(29, -1, -1):
        b, e = _dist_base(c)
        if b <= d:
            return c, e, d - b


def fixed_tokens(bw, toks, final=True):
    """One fixed block of tokens: ints are literals, (length, distance) matches; raw ('L', sym) / ('D', sym) emit a symbol."""
    lit = canon([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
    bw.put(1 if final else 0, 1)
    bw.put(1, 2)
    for t in toks:
        if isinstance(t, int):
            bw.code(*lit[t])
        elif t[0] == "L":
            bw.code(*lit[t[1]])
        elif t[0] == "D":
            bw.code(t[1], 5)
        else:
            s, e, x = len_sym(t[0])
            bw.code(*lit[s])
            bw.put(x, e)
            ds, de, dx = dist_sym(t[1])
            bw.code(ds, 5)
            bw.put(dx, de)
    bw.code(*lit[256])


def dynamic_header(bw, lit_lens, dist_lens, final=True, hlit=None, hdist=None, cl_syms=None, cl_lens=None):
    """Dynamic block header. Code lengths are sent as symbols 0..15 with a complete 4-bit code-length code, unless cl_syms
    ([(sym, extra bits value)]) and cl_lens (19 code-length code lengths) are given."""
    bw.put(1 if final else 0, 1)
    bw.put(2, 2)
    bw.put((len(lit_lens) if hlit is None else hlit) - 257, 5)
    bw.put((len(dist_lens) if hdist is None else hdist) - 1, 5)
    if cl_lens is None:
        cl_lens = [4] * 16 + [0, 0, 0]
    bw.put(19 - 4, 4)
    for k in range(19):
        bw.put(cl_lens[ORDER[k]], 3)
    clc = canon(cl_lens)
    if cl_syms is None:
        cl_syms = [(v, 0) for v in list(lit_lens) + list(dist_lens)]
    for s, x in cl_syms:
        bw.code(*clc[s])
        if s >= 16:
            bw.put(x, {16: 2, 17: 3, 18: 7}[s])


def dynamic_body(bw, lit_lens, dist_lens, toks):
    lit, dist = canon(lit_lens), canon(dist_lens)
    for t in toks:
        if isinstance(t, int):
            bw.code(*lit[t])
        else:
            s, e, x = len_sym(t[0])
            bw.code(*lit[s])
            bw.put(x, e)
            ds, de, dx = dist_sym(t[1])
            bw.code(*dist[ds])
            bw.put(dx, de)
    bw.code(*lit[256])


def finish(bw, payload, header=b"\x78\x01"):
    bw.align()
    return header + bytes(bw.o) + zlib.adler32(payload).to_bytes(4, "big")


def level0(p):
    """fast_level0_compress's layout: 78 01, stored blocks of <= 65535 bytes, Adler-32."""
    o = bytearray(b"\x78\x01")
    at = 0
    while True:
        n = min(65535, len(p) - at)
        last = at + n == len(p)
        o += bytes([1 if last else 0]) + n.to_bytes(2, "little") + (n ^ 0xffff).to_bytes(2, "little") + p[at:at + n]
        at += n
        if last:
            break
    return bytes(o) + zlib.adler32(p).to_bytes(4, "big")


def lit_lens_with(used, extra=()):
    """A complete literal/length code: the `used` literals, EOB, and the `extra` length symbols."""
    syms = sorted(set(used) | {256} | set(extra))
    n = len(syms)
    L = (n - 1).bit_length()
    lo = (1 << L) - n   # lo symbols of length L - 1 and n - lo of length L: sum 2^-len == 1
    lens = [0] * 286
    for i, s in enumerate(syms):
        lens[s] = L - 1 if i < lo else L
    return lens


def handmade():
    """[(name, stream, payload)] of valid hand-made streams."""
    out = []
    rng = np.random.default_rng(11)
    # distance 32768 and length 258 in a fixed block
    head = rng.integers(0, 256, size=300, dtype=np.uint8).tobytes()
    fill = bytes(range(97, 123)) * ((32768 - 300) // 26 + 1)
    fill = fill[:32768 - 300]
    p = head + fill + head
    bw = BitW()
    tk = list(head) + list(fill[:26])
    left = len(fill) - 26
    while left > 0:
        piece = 258 if left >= 261 or left == 258 else (left - 3 if left > 258 else left)
        tk.append((piece, 26))
        left -= piece
    tk += [(258, 32768), (42, 32768)]
    fixed_tokens(bw, tk)
    out.append(("dist_32768", finish(bw, p), p))
    # a dynamic block with no distance code at all (HDIST = 1, length 0): literals only
    p = b"dynamic block without distances " * 4
    lens = lit_lens_with(used=set(p))
    bw = BitW()
    dynamic_header(bw, lens, [0])
    dynamic_body(bw, lens, [0], list(p))
    out.append(("no_dist_code", finish(bw, p), p))
    # a single distance code of length 1 (incomplete, accepted), used by a match at distance 1..: symbol 3 -> distance 4
    p = b"abcd" * 40
    lens = lit_lens_with(used=set(b"abcd"), extra=[len_sym(156)[0]])
    dl = [0, 0, 0, 1]
    bw = BitW()
    dynamic_header(bw, lens, dl)
    dynamic_body(bw, lens, dl, list(b"abcd") + [(156, 4)])
    out.append(("single_dist_code", finish(bw, p), p))
    # code-length repeats 16 / 17 / 18 with a code-length code over 0, 8, 16, 17, 18
    p = bytes(range(256)) * 2
    lens = [8] * 254 + [9, 9] + [8] + [0] * 29   # literals 0..253 and EOB of 8 bits, 254 / 255 of 9: complete
    dlens = DL
    cl_lens = [0] * 19
    cl_lens[8] = 2
    cl_lens[9] = cl_lens[4] = cl_lens[5] = cl_lens[16] = cl_lens[17] = cl_lens[18] = 3
    syms = [(8, 0), (16, 3), (16, 3), (16, 3), (16, 3)]          # 1 + 4 * 6 = 25 eights
    n8 = 25
    while n8 + 6 <= 254:
        syms.append((16, 3))
        n8 += 6
    syms += [(8, 0)] * (254 - n8)
    syms += [(9, 0), (9, 0), (8, 0)]                               # 254, 255, 256
    syms += [(17, 7 - 3)]                                          # 7 zeros: 257..263
    syms += [(18, 22 - 11)]                                        # 22 zeros: 264..285
    syms += [(5, 0), (16, 3), (16, 3), (16, 3), (16, 3), (16, 0), (4, 0), (4, 0)]   # 1 + 24 + 3 fives, 2 fours
    bw = BitW()
    dynamic_header(bw, lens, dlens, cl_syms=syms, cl_lens=cl_lens)
    dynamic_body(bw, lens, dlens, list(p))
    out.append(("cl_repeats", finish(bw, p), p))
    return out


def payloads():
    rng = np.random.default_rng(20261017)
    rnd = lambda n: rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    words = [b"micro", b"block", b"header", b"column", b"scan", b"offset", b"the", b"of", b"zlib", b"sstable"]
    text = lambda n: b" ".join(words[i] for i in rng.integers(0, len(words), size=n))
    # symbol counts growing by 1.7x: a Huffman tree 15 deep (Fibonacci counts tie, and zlib breaks ties toward shallow trees)
    w = [1]
    for k in range(1, 16):
        w.append(max(int(round(1.7 ** k)), w[-1] + 1))
    skew = bytes(np.repeat(np.arange(16, dtype=np.uint8) * 7 + 1, w)[rng.permutation(sum(w))])
    out = [b"", b"a", rnd(7), rnd(200), bytes(255), bytes(300), rnd(1000), rng.integers(0, 16, size=3000, dtype=np.uint8).tobytes(),
           text(800), text(1500), np.cumsum(rng.integers(0, 100, size=1000)).astype(np.int64).tobytes(),
           rng.integers(0, 40, size=2000).astype(np.int64).tobytes(), bytes(70_000), text(12_000), skew,
           rnd(20) + rnd(258) * 3 + rnd(20)]
    for d in (1, 3, 17, 1000):                                  # repeats at distance d
        pat = rnd(d)
        out.append(rnd(20) + pat * (2 + 3000 // d) + rnd(20))
    return out


def flushed(p, modes):
    """Stream of p with the given flush modes between equal parts (empty stored blocks at sync / full flushes)."""
    c = zlib.compressobj(6)
    parts = np.array_split(np.frombuffer(p, dtype=np.uint8), len(modes) + 1)
    o = b""
    for part, m in zip(parts, modes):
        o += c.compress(part.tobytes()) + c.flush(m)
    return o + c.compress(parts[-1].tobytes()) + c.flush()


def malformed(streams, rng):
    """[(stream, payload index, refusal name it is built to reach, strict name)]"""
    bad = []
    # truncations and one-bit flips of the small streams
    for s, i, _ in streams:
        if len(s) > 3000:
            continue
        for cut in sorted({len(s) - 1, len(s) // 2, 1}):
            bad.append((s[:cut], i, "truncated", ""))
        for at in sorted(set(rng.integers(2, len(s), size=min(6, len(s) - 2)).tolist())):
            t = bytearray(s)
            t[at] ^= 1 << int(rng.integers(0, 8))
            bad.append((bytes(t), i, "", ""))
    return bad


def handmade_bad(pays):
    """[(stream, payload bytes, refusal)]: one or more streams per refusal branch."""
    out = []
    p = b"hello hello hello zlib"
    good = compress(p, 6)
    body = good[2:]
    hdr = lambda cmf, flg: bytes([cmf, flg + (31 - (cmf * 256 + flg) % 31) % 31])   # FCHECK made right
    out.append((hdr(0x79, 0x80) + body, p, "header_cm"))                         # CM 9
    out.append((hdr(0x88, 0x80) + body, p, "header_cinfo"))                      # CINFO 8
    out.append((b"\x78\x9d" + body, p, "header_fcheck"))
    out.append((hdr(0x78, 0xa0) + b"\0\0\0\1" + body, p, "fdict"))              # FDICT, a DICTID
    out.append((b"\x78\x01\x07" + bytes(8), p, "btype3"))                      # BFINAL 1, BTYPE 3
    st = level0(p)
    t = bytearray(st)
    t[5] ^= 1                                                                   # NLEN
    out.append((bytes(t), p, "stored_nlen"))
    # dynamic headers
    lens = lit_lens_with(used=set(p))
    for hlit, name in ((287, "hlit"), (288, "hlit")):
        bw = BitW()
        dynamic_header(bw, lens + [0] * (hlit - 286), DL, hlit=hlit)
        out.append((finish(bw, p), p, name))
    for hdist in (31, 32):
        bw = BitW()
        dynamic_header(bw, lens, [5] * hdist, hdist=hdist)
        out.append((finish(bw, p), p, "hdist"))
    cl_rep = [0] * 19
    for s in (0, 5, 16, 17, 18):
        cl_rep[s] = 3
    cl_rep[0], cl_rep[5] = 2, 2      # 2 * 1/4 + 3 * 1/8 = 7/8: incomplete -- make 16 length 2
    cl_rep[16] = 2
    cl_rep[17] = cl_rep[18] = 3      # 3/4 + 2/8 = 1
    bw = BitW()
    dynamic_header(bw, lens, DL, cl_syms=[(16, 0)] + [(0, 0)] * 313, cl_lens=cl_rep)
    out.append((finish(bw, p), p, "repeat_first"))
    bw = BitW()
    dynamic_header(bw, lens, DL, cl_syms=[(18, 127)] * 3, cl_lens=cl_rep)   # 3 x 138 zeros > 316
    out.append((finish(bw, p), p, "run_past"))
    over = list(lens)
    over[[s for s in range(286) if over[s]][0]] -= 1                            # one code shorter: over-subscribed
    bw = BitW()
    dynamic_header(bw, over, DL)
    out.append((finish(bw, p), p, "oversubscribed"))
    bw = BitW()
    dynamic_header(bw, lens, DL, cl_lens=[4] * 15 + [0] * 4)              # 15 * 1/16: incomplete code-length code
    out.append((finish(bw, p), p, "incomplete_cl"))
    inc = list(lens)
    inc[min(s for s in range(286) if inc[s])] = 0
    bw = BitW()
    dynamic_header(bw, inc, DL)
    out.append((finish(bw, p), p, "incomplete_lit"))
    bw = BitW()
    dynamic_header(bw, lens, [5] * 29 + [0])                                    # 29 codes of 5 bits
    out.append((finish(bw, p), p, "incomplete_dist"))
    bw = BitW()
    dynamic_header(bw, lens, [2, 2])                                            # two distance codes of length 2
    out.append((finish(bw, p), p, "incomplete_dist"))
    noeob = list(lens)
    noeob[256] = 0
    bw = BitW()
    dynamic_header(bw, noeob, DL)
    out.append((finish(bw, p), p, "missing_eob"))
    # fixed-block symbols and distances
    for sym in (286, 287):
        bw = BitW()
        fixed_tokens(bw, list(p[:4]) + [("L", sym), ("D", 0)])
        out.append((finish(bw, p), p, "lit_286"))
    for ds in (30, 31):
        bw = BitW()
        fixed_tokens(bw, list(p[:4]) + [("L", 257), ("D", ds)])
        out.append((finish(bw, p), p, "dist_30"))
    bw = BitW()
    fixed_tokens(bw, list(p[:4]) + [(3, 5)])
    out.append((finish(bw, p), p, "dist_too_far"))
    bw = BitW()
    fixed_tokens(bw, [(3, 1)])
    out.append((finish(bw, p), p, "dist_too_far"))
    out.append((good[:-1] + bytes([good[-1] ^ 1]), p, "adler"))
    out.append((compress(p + b"!", 6), p, "output_long"))
    out.append((compress(p[:-1], 6), p, "output_short"))
    out.append((good[:-2], p, "truncated"))
    out.append((good + b"\0", p, "trailing_bytes"))
    out.append((good + good, p, "trailing_bytes"))
    return out


def main():
    z = libz()
    assert z is not None, "libz.so.1 is required to make the vectors"
    pays = payloads()
    streams = []   # (stream, payload index, kind)
    kinds = ["level", "strategy", "flush", "level0", "handmade"]
    for i, p in enumerate(pays):
        for lv in (0, 1, 6, 9):
            streams.append((compress(p, lv), i, 0))
        for strat in (zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED):
            streams.append((compress(p, 6, strat), i, 1))
    for i in (9, 13, 12):
        streams.append((flushed(pays[i], [zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH, zlib.Z_SYNC_FLUSH]), i, 2))
    streams.append((compress(pays[9], 6, wbits=9), 9, 0))                    # CINFO 1
    big = b"".join(pays[k] for k in (9, 13, 12, 8))                          # > 65535: several stored blocks
    pays.append(big)
    streams.append((level0(big), len(pays) - 1, 3))
    streams.append((level0(pays[2]), 2, 3))
    for _, s, p in handmade():
        pays.append(p)
        streams.append((s, len(pays) - 1, 4))
    for s, i, _ in streams:
        assert uncompress(z, s, len(pays[i])) == pays[i], i
        assert walk(s)[0] == pays[i], i
    census = np.zeros((len(streams), len(CENSUS)), dtype=np.uint8)
    for k, (s, _, _) in enumerate(streams):
        for name in walk(s)[1] - {"trailing"}:
            census[k, CENSUS.index(name)] = 1
    rng = np.random.default_rng(7)
    bad = [(s, i, REFUSALS.index(r), STRICT.index(st)) for s, i, r, st in malformed(streams, rng)]
    for s, p, r in handmade_bad(pays):
        if p not in pays:
            pays.append(p)
        bad.append((s, pays.index(p), REFUSALS.index(r), 1 if r == "trailing_bytes" else 0))
    for s, i, r, _ in bad:   # the hand-made streams reach the branch they are named after
        if r and REFUSALS[r] not in ("trailing_bytes", "output_long", "output_short"):
            try:
                walk(s)
                raise AssertionError(("accepted", REFUSALS[r]))
            except Bad as e:
                assert str(e) == REFUSALS[r], (str(e), REFUSALS[r])
    outs = [uncompress(z, s, len(pays[i])) for s, i, _, _ in bad]
    verdict = np.array([o is not None for o in outs], dtype=np.uint8)
    digest = np.array([np.frombuffer(hashlib.sha256(o).digest() if o is not None else bytes(32), dtype=np.uint8) for o in outs])
    cat = lambda bs: (np.frombuffer(b"".join(bs), dtype=np.uint8),
                      np.concatenate([[0], np.cumsum([len(b) for b in bs])]).astype(np.int64))
    pay, pay_off = cat(pays)
    st, st_off = cat([s for s, _, _ in streams])
    bd, bd_off = cat([s for s, _, _, _ in bad])
    np.savez_compressed(os.path.join(HERE, "zlib_vectors.npz"), payloads=pay, payload_off=pay_off, streams=st, stream_off=st_off,
                        stream_payload=np.array([i for _, i, _ in streams], dtype=np.int32),
                        stream_kind=np.array([k for _, _, k in streams], dtype=np.int32), kinds=np.array(kinds),
                        bad=bd, bad_off=bd_off, bad_payload=np.array([i for _, i, _, _ in bad], dtype=np.int32),
                        bad_refusal=np.array([r for _, _, r, _ in bad], dtype=np.int32), refusal_names=np.array(REFUSALS),
                        bad_strict=np.array([s for _, _, _, s in bad], dtype=np.int32), strict_names=np.array(STRICT),
                        bad_zlib_ok=verdict, bad_zlib_sha256=digest, census=census, census_names=np.array(CENSUS),
                        zlib_version=np.array(z.zlibVersion().decode()))
    miss = [CENSUS[j] for j in range(len(CENSUS)) if not census[:, j].any()]
    print(f"{len(pays)} payloads, {len(streams)} streams, {len(bad)} malformed ({int(verdict.sum())} accepted by zlib), "
          f"zlib {z.zlibVersion().decode()}, census misses {miss}, {os.path.getsize(os.path.join(HERE, 'zlib_vectors.npz'))} bytes")


if __name__ == "__main__":
    main()
