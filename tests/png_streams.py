"""PNG files whose zlib streams probe the GPU inflate where zlib, as PIL drives it, decides: every zlib error rule placed before
the image's end, after it in the same read and after it past an IDAT boundary; images that end on a literal or a match at and
around PIL's 64 KiB read boundaries and across IDAT splits; and streams over several speculative chunks.  Each case is
(name, file); oracle/inflate_ref.py gives what PIL makes of it and what the status words must be."""
from __future__ import annotations

import zlib
from typing import List, Tuple

import numpy as np

from oracle import deflate_ref as D
from png_cases import filter_rows, png_file, random_rows

W, H = 20, 6                   # the small grey image the error rules ride on
ROW = W + 1


def _raw(rng, w=W, h=H, content="photo"):
    return filter_rows(random_rows(rng, w, h, 0, 8, content), 1, (0, 1, 2, 3, 4))


def _end(w: D.BitWriter, data: bytes, tail: bytes = b"") -> bytes:
    """The zlib stream of the image `data`: header 78 01, the blocks, then `tail` (padding or a stand-in Adler-32)."""
    return b"\x78\x01" + w.getvalue() + tail


# --- zlib's error rules, each as the blocks that break it (written at the writer's position) -------------------------------

def _cl(**lens):
    cl = [0] * 19
    for k, v in lens.items():
        cl[int(k[1:])] = v
    return cl


def _rule_writers():
    """(name, writer(w)) for every rule: the writer puts the blocks that break it at the writer's position."""
    fixed_codes = D.canonical(D.FIXED_LIT)

    def stored_bad(w):
        w.bits(0, 3)
        w.align()
        w.bits(5, 16)
        w.bits(5, 16)

    def hdr(nlen, ndist):
        return lambda w: D.dynamic_header(w, False, nlen, ndist, _cl(s0=1, s1=1), [], ncode=4)

    def lit_set(lengths_cl, lengths):
        return lambda w: D.dynamic_header(w, False, 257, 1, lengths_cl, lengths)

    rules = [
        ("block type 3", lambda w: w.bits(0b110, 3)),
        ("LEN != ~NLEN", stored_bad),
        ("HLIT 287", hdr(287, 1)), ("HLIT 288", hdr(288, 1)), ("HDIST 31", hdr(257, 31)), ("HDIST 32", hdr(257, 32)),
        ("incomplete code-length code", lambda w: D.dynamic_header(w, False, 257, 1, _cl(s0=1), [], ncode=4)),
        ("over-subscribed code-length code", lambda w: D.dynamic_header(w, False, 257, 1, _cl(s0=1, s1=1, s2=1), [], ncode=19)),
        ("all-zero code-length code", lambda w: D.dynamic_header(w, False, 257, 1, [0] * 19, [], ncode=4)),
        ("repeat 16 first", lambda w: D.dynamic_header(w, False, 257, 1, _cl(s0=1, s16=1), [(16, 0)])),
        ("repeat past HLIT + HDIST", lambda w: D.dynamic_header(w, False, 257, 1, _cl(s0=1, s18=1), [(18, 127), (18, 127)])),
        ("no end-of-block code", lit_set(_cl(s0=1, s1=2, s18=2), [1, 1, (18, 127), (18, 107)])),
        ("over-subscribed literal code", lit_set(_cl(s0=1, s1=2, s18=2), [1, 1, (18, 127), (18, 105), 1, 0])),
        ("incomplete literal code of several codes", lit_set(_cl(s0=1, s1=2, s2=3, s18=3), [1, (18, 127), (18, 106), 2, 0])),
    ]

    def fixed_lit(sym):
        def f(w):
            w.bits(0b010, 3)
            w.code(fixed_codes[sym], D.FIXED_LIT[sym])
        return f

    def fixed_dist(sym):
        def f(w):
            w.bits(0b010, 3)
            w.code(fixed_codes[257], 7)       # length 3
            w.bits(int(format(sym, "05b")[::-1], 2), 5)
        return f

    def empty_dist(w):
        lit = [0] * 258
        lit[0] = lit[256] = lit[257] = 2
        lit[1] = 2
        D.dynamic_header(w, False, 258, 1, _cl(s0=1, s2=1), [2, 2] + [0] * 254 + [2, 2, 0])
        D.tokens_with(w, [1, (3, 1)], lit, [0])

    rules += [("literal code 286 in a fixed block", fixed_lit(286)), ("literal code 287 in a fixed block", fixed_lit(287)),
              ("distance code 30 in a fixed block", fixed_dist(30)), ("distance code 31 in a fixed block", fixed_dist(31)),
              ("length code behind an empty distance tree", empty_dist)]
    return rules


def error_rule_cases(seed: int = 21) -> List[Tuple[str, str, bytes]]:
    """(rule, placement, file) for every zlib error rule at three places: "before" (inside the image), "same read" (after the
    image in the read that completed it), "next IDAT" (after the image, past an IDAT boundary).  The image is one non-final
    fixed block of literals; an empty stored block after it byte-aligns what follows."""
    rng = np.random.default_rng(seed)
    raw = _raw(rng)
    out = []
    rules = _rule_writers()
    for name, rule in rules:
        # before the image's end: half the image, then the rule, then padding
        w = D.BitWriter()
        D.fixed(w, list(raw[:len(raw) // 2]), False)
        rule(w)
        out.append((name, "before", png_file(W, H, 0, 8, _end(w, raw, bytes(48)))))
        # after the image
        w = D.BitWriter()
        D.fixed(w, list(raw), False)
        done = 2 + (w.tell() - 7 + 7) // 8          # stream bytes up to the image's last bit (before the 7-bit end-of-block)
        D.stored(w, b"", False)
        rule(w)
        z = _end(w, raw, bytes(48))
        out.append((name, "same read", png_file(W, H, 0, 8, z)))
        out.append((name, "next IDAT", png_file(W, H, 0, 8, z, split=[done])))
    # a distance before the stream's start, and a bad Adler-32
    w = D.BitWriter()
    D.fixed(w, [7, (3, 5)] + list(raw[4:]), True)
    out.append(("distance before the stream", "before", png_file(W, H, 0, 8, D.zlib_wrap(w.getvalue(), raw))))
    w = D.BitWriter()
    D.fixed(w, list(raw), False)
    done = 2 + (w.tell() - 7 + 7) // 8
    D.fixed(w, [(3, len(raw) + 5)], True)
    z = D.zlib_wrap(w.getvalue(), raw)
    out += [("distance before the stream", "same read", png_file(W, H, 0, 8, z)),
            ("distance before the stream", "next IDAT", png_file(W, H, 0, 8, z, split=[done]))]
    bad = zlib.compress(raw[:3 * ROW])
    out.append(("bad Adler-32", "before", png_file(W, H, 0, 8, bad[:-1] + bytes([bad[-1] ^ 1]))))
    z = zlib.compress(raw)
    z = z[:-1] + bytes([z[-1] ^ 1])
    out += [("bad Adler-32", "same read", png_file(W, H, 0, 8, z)),
            ("bad Adler-32", "next IDAT", png_file(W, H, 0, 8, z, split=[len(z) - 4]))]
    out += [(n, "last bits", f) for n, f in last_bits_cases(raw)]
    return out


def last_bits_cases(raw: bytes) -> List[Tuple[str, bytes]]:
    """An invalid code in the stream's last 1..14 bits: the image complete in a non-final fixed block, then a final dynamic
    block whose literal/length code is the one-bit code of end-of-block, led by the bit 1 that is no code (or a length code
    behind a one-code distance tree, led by the distance bit 1), and nothing after it but zero padding (no Adler-32)."""
    out = []
    for k in range(1, 15):
        for kind in ("literal", "distance"):
            for shift, ncode in [(s, n) for s in range(16) for n in (18, 19)]:
                w = D.BitWriter()
                D.fixed(w, list(raw), False)
                for _ in range(shift):
                    D.fixed(w, [], False)         # 10 bits each: moves where the last block starts
                if kind == "literal":
                    lit = [0] * 257
                    lit[256] = 1
                    D.dynamic_header(w, True, 257, 1, _cl(s0=1, s1=1), lit + [0], ncode=ncode)
                else:
                    lit = [0] * 258
                    lit[256] = lit[257] = 1
                    D.dynamic_header(w, True, 258, 1, _cl(s0=1, s1=1), lit + [1], ncode=ncode)
                    w.bits(1, 1)                  # length code 257
                start = w.tell()
                w.bits(1, 1)
                pad = k - 1 - (-(w.tell()) % 8)
                if pad < 0 or pad % 8:
                    continue
                data = w.getvalue() + bytes(pad // 8)
                assert 8 * len(data) - start == k
                out.append((f"invalid {kind} code in the last {k} bits", png_file(W, H, 0, 8, b"\x78\x01" + data)))
                break
    return out


# --- where the image ends ---------------------------------------------------------------------------------------------

def _image_block(kind: str, raw: bytes):
    """Tokens of the image ending on a literal, on a match that ends exactly at the image's end, or on one that runs past it."""
    if kind == "literal":
        return list(raw)
    if kind == "match to the end":
        return list(raw[:-ROW]) + [(ROW, ROW)] if raw[-ROW:] == raw[-2 * ROW:-ROW] else None
    return list(raw[:-ROW]) + [(ROW + 40, ROW)]


def _repeating_raw(rng):
    rows = np.tile(random_rows(rng, W, 1, 0, 8, "noise"), (H, 1))
    return filter_rows(rows, 1, (0,))


def image_end_cases(seed: int = 22, ks=(1, 2, 5)) -> List[Tuple[str, bytes]]:
    """The image's last bit at stream byte 65536k - 2, 65536k - 1 and 65536k (the read ends after 65536k - 1), with an invalid
    block type right behind the image, for each way the image ends; empty stored blocks fill the stream up to there.  Then the
    same images over one-byte IDATs, empty IDATs and an Adler-32 split across IDATs."""
    rng = np.random.default_rng(seed)
    raw = _repeating_raw(rng)
    out = []
    for kind in ("literal", "match to the end", "match past the end"):
        toks = _image_block(kind, raw)
        for k in ks:
            for delta in (-1, 0, 1):
                target = 65536 * k - 1 + delta          # stream byte that holds the image's last bit
                def blocks(m, s1, s2):
                    """m empty stored blocks, s1 empty fixed blocks, an empty stored block, s2 empty fixed blocks, the image"""
                    w = D.BitWriter()
                    for _ in range(m):
                        D.stored(w, b"", False)
                    for _ in range(s1):
                        D.fixed(w, [], False)
                    D.stored(w, b"", False)
                    for _ in range(s2):
                        D.fixed(w, [], False)
                    D.fixed(w, toks, False)
                    return w, 2 + (w.tell() - 7 - 1) // 8    # the last token's last bit, before the 7-bit end-of-block
                s1, s2 = next((s1, s2) for s1 in range(8) for s2 in range(8) if (target - blocks(0, s1, s2)[1]) % 5 == 0)
                w, byte = blocks((target - blocks(0, s1, s2)[1]) // 5, s1, s2)
                assert byte == target
                w.bits(0b110, 3)                    # block type 3
                z = _end(w, raw, bytes(4))
                out.append((f"{kind}, last bit at 65536*{k}{delta - 1:+d}", png_file(W, H, 0, 8, z)))
        w = D.BitWriter()
        D.fixed(w, toks, True)
        z = D.zlib_wrap(w.getvalue(), raw)
        out += [(f"{kind}, one-byte IDATs", png_file(W, H, 0, 8, z, split=list(range(1, len(z))))),
                (f"{kind}, empty IDATs", png_file(W, H, 0, 8, z, split=[0, 0, 3, 3, len(z) - 4, len(z) - 4, len(z), len(z)])),
                (f"{kind}, Adler-32 split across IDATs", png_file(W, H, 0, 8, z, split=[len(z) - 3, len(z) - 1]))]
        for bad_tail in (1, 3):
            zb = z[:-1] + bytes([z[-1] ^ 1])
            out.append((f"{kind}, bad Adler-32 split {bad_tail} from the end", png_file(W, H, 0, 8, zb, split=[len(z) - bad_tail])))
    return out


# --- streams over several speculative chunks ---------------------------------------------------------------------------

def _long_literal_code():
    """Literal/length code lengths with every literal 15 bits long (end-of-block and six length codes take the rest): 64 KiB
    of such literals inflate to about 35 KiB, so the chunks' outputs are short."""
    lit = [15] * 256 + [1, 2, 3, 4, 5, 6, 7]
    return lit + [0] * (286 - len(lit))


def multi_chunk_cases(seed: int = 23) -> List[Tuple[str, bytes]]:
    rng = np.random.default_rng(seed)
    out = []
    # one dynamic block over several chunks
    raw = filter_rows(random_rows(rng, 399, 400, 0, 8, "photo"), 1, (1, 2, 4))
    w = D.BitWriter()
    D.dynamic(w, list(raw), True)
    out.append(("one dynamic block over several chunks", png_file(399, 400, 0, 8, D.zlib_wrap(w.getvalue(), raw))))
    # short chunks (blocks of 64 fifteen-bit literals), then matches at distance 32768 whose sources reach back over them and
    # straddle their starts; rows of 256 bytes keep the filter bytes in place
    rows1, rows2 = 200, 130
    first = filter_rows(random_rows(rng, 255, rows1, 0, 8, "photo"), 1, (0, 1, 2, 3, 4))
    raw = bytearray(first)
    for i in range(256 * rows2):
        raw.append(raw[-32768])
    raw = bytes(raw)
    lit = _long_literal_code()
    w = D.BitWriter()
    for k in range(0, len(first), 64):
        D.dynamic(w, list(first[k:k + 64]), False, lit_lens=lit, dist_lens=[0])
    D.fixed(w, [(258, 32768)] * (256 * rows2 // 258) + [(256 * rows2 % 258, 32768)], True)
    out.append(("distance 32768 back over short chunks", png_file(255, rows1 + rows2, 0, 8, D.zlib_wrap(w.getvalue(), raw))))
    # a chunk whose output overflows its capacity: photo rows, then 2000 rows of zeros, then photo rows
    rows = np.concatenate([random_rows(rng, 299, 300, 0, 8, "photo"), np.zeros((2000, 299), np.uint8),
                           random_rows(rng, 299, 200, 0, 8, "noise")])
    raw = filter_rows(rows, 1, (0,))
    out.append(("a chunk over its symbol capacity", png_file(299, 2500, 0, 8, zlib.compress(raw, 6))))
    # a false candidate: a stored block whose data holds a zlib stream's dynamic header, across chunk 1's start, before the
    # true block boundaries
    a = filter_rows(random_rows(rng, 255, 300, 0, 8, "photo"), 1, (1,))
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    head = co.compress(a[:64000]) + co.flush(zlib.Z_SYNC_FLUSH)
    fake = zlib.compress(a[64000:], 9)[2:2000]
    assert len(head) < 65536 - 200
    f = 65536 + 100 - 2 - len(head) - 5                   # stored data up to just past chunk 1's start
    f += (1 - f) % 256                                      # the copied header starts just after a row's filter byte
    stored_data = bytearray(bytes(f) + fake)
    stored_data[::256] = bytes(len(stored_data[::256]))     # filter bytes 0
    stored_data = bytes(stored_data)
    rest = a[64000:]
    co2 = zlib.compressobj(6, zlib.DEFLATED, -15)
    tail = co2.compress(rest) + co2.flush()
    # the image: a's first 64000 bytes, the stored data, then the rest of a, in rows of 256 (the stored data pads to rows)
    pad = (-len(stored_data)) % 256
    w2 = D.BitWriter()
    D.stored(w2, stored_data + bytes(pad), False)
    raw = a[:64000] + stored_data + bytes(pad) + rest
    body = head + w2.getvalue() + tail
    assert len(raw) % 256 == 0
    out.append(("false candidate before the true block boundaries",
                png_file(255, len(raw) // 256, 0, 8, b"\x78\x01" + body + zlib.adler32(raw).to_bytes(4, "big"))))
    # zlib's own streams: stored (level 0, noise), dynamic and fixed-Huffman
    noise = filter_rows(random_rows(rng, 300, 300, 2, 8, "noise"), 3, (0,))
    photo = filter_rows(random_rows(rng, 400, 300, 2, 8, "photo"), 3, (1, 2, 3, 4))
    out += [("zlib level 0", png_file(300, 300, 2, 8, zlib.compress(noise, 0))),
            ("noise at zlib level 6", png_file(300, 300, 2, 8, zlib.compress(noise, 6))),
            ("photo at zlib level 6", png_file(400, 300, 2, 8, zlib.compress(photo, 6))),
            ("photo, fixed Huffman only", png_file(400, 300, 2, 8, _zlib(photo, zlib.Z_FIXED)))]
    return out


def _zlib(data: bytes, strategy: int) -> bytes:
    co = zlib.compressobj(6, zlib.DEFLATED, 15, 9, strategy)
    return co.compress(data) + co.flush()
