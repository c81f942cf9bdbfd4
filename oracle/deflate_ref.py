"""A raw DEFLATE writer (RFC 1951) for streams zlib never emits, and zlib framing (RFC 1950).

A stream is built from blocks; each block holds tokens: an int (a literal byte) or a tuple (length, distance) for a match.
``stored`` / ``fixed`` / ``dynamic`` write one block each; ``dynamic`` takes explicit code lengths, so tests can make one-code and
empty distance codes, 15-bit codes and other shapes zlib's encoder does not choose.  ``dynamic_header`` writes a dynamic block's
header field by field (HLIT 287 / 288, HDIST 31 / 32, any code-length code, any repeat), for headers zlib must refuse.
``BitWriter.tell`` gives the bit a block starts at.  ``zlib_wrap`` adds the header and Adler-32.
"""
from __future__ import annotations

import zlib
from typing import List, Optional, Sequence, Tuple, Union

Token = Union[int, Tuple[int, int]]

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
         12289, 16385, 24577]
DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
VIA_284 = "via284"      # a match token (258, dist, VIA_284) writes length 258 as code 284 with all five extra bits set


class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def bits(self, value: int, count: int) -> None:
        """`count` bits of `value`, least significant first."""
        self.acc |= (value & ((1 << count) - 1)) << self.n
        self.n += count
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def code(self, code: int, length: int) -> None:
        """A Huffman code, most significant bit first."""
        for i in range(length - 1, -1, -1):
            self.bits((code >> i) & 1, 1)

    def align(self) -> None:
        if self.n:
            self.bits(0, 8 - self.n)

    def tell(self) -> int:
        """Bits written so far: the position of the next bit in the raw DEFLATE stream."""
        return 8 * len(self.out) + self.n

    def getvalue(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lengths: Sequence[int]) -> List[int]:
    """RFC 1951 3.2.2: the codes of a canonical Huffman code with these lengths."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lengths:
        out.append(nxt[l] if l else 0)
        if l:
            nxt[l] += 1
    return out


def huffman_lengths(freq: Sequence[int], limit: int = 15) -> List[int]:
    """Code lengths for symbol frequencies (every used symbol gets a code; at least two codes), at most `limit` bits."""
    import heapq
    used = [i for i, f in enumerate(freq) if f]
    if len(used) < 2:
        used = (used + [i for i in range(len(freq)) if i not in used])[:2]
    lengths = [0] * len(freq)
    heap = [(max(freq[i], 1), [i]) for i in used]
    heapq.heapify(heap)
    while len(heap) > 1:
        fa, a = heapq.heappop(heap)
        fb, b = heapq.heappop(heap)
        for s in a + b:
            lengths[s] += 1
        heapq.heappush(heap, (fa + fb, a + b))
    if max(lengths) > limit:     # flatten: a complete code of equal-ish lengths over the used symbols
        k = len(used)
        bits = (k - 1).bit_length()
        short = (1 << bits) - k      # codes of bits - 1
        for j, s in enumerate(used):
            lengths[s] = bits - 1 if j < short else bits
    return lengths


def _length_symbol(length: int, via284: bool = False) -> Tuple[int, int, int]:
    if via284:
        return 284, 31, 5
    if length == 258:
        return 285, 0, 0
    for i in range(28, -1, -1):
        if LBASE[i] <= length and i != 28:
            return 257 + i, length - LBASE[i], LEXT[i]
    raise ValueError(length)


def _dist_symbol(dist: int) -> Tuple[int, int, int]:
    for i in range(29, -1, -1):
        if DBASE[i] <= dist:
            return i, dist - DBASE[i], DEXT[i]
    raise ValueError(dist)


def _symbols(tokens: Sequence[Token]):
    for t in tokens:
        if isinstance(t, int):
            yield t, None
        else:
            yield _length_symbol(t[0], len(t) > 2 and t[2] == VIA_284), _dist_symbol(t[1])


def _write_tokens(w: BitWriter, tokens, lit_codes, lit_lens, dist_codes, dist_lens) -> None:
    for lit, dist in _symbols(tokens):
        if dist is None:
            w.code(lit_codes[lit], lit_lens[lit])
            continue
        sym, extra, nb = lit
        w.code(lit_codes[sym], lit_lens[sym])
        w.bits(extra, nb)
        dsym, dextra, dnb = dist
        w.code(dist_codes[dsym], dist_lens[dsym])
        w.bits(dextra, dnb)
    w.code(lit_codes[256], lit_lens[256])


def stored(w: BitWriter, data: bytes, final: bool) -> None:
    """One stored block (at most 65535 bytes)."""
    assert len(data) <= 65535
    w.bits(int(final), 1)
    w.bits(0, 2)
    w.align()
    w.bits(len(data), 16)
    w.bits(len(data) ^ 0xFFFF, 16)
    for b in data:
        w.bits(b, 8)


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def fixed(w: BitWriter, tokens: Sequence[Token], final: bool) -> None:
    w.bits(int(final), 1)
    w.bits(1, 2)
    _write_tokens(w, tokens, canonical(FIXED_LIT), FIXED_LIT, canonical(FIXED_DIST), FIXED_DIST)


def dynamic(w: BitWriter, tokens: Sequence[Token], final: bool, lit_lens: Optional[Sequence[int]] = None,
            dist_lens: Optional[Sequence[int]] = None, cl_lens: Optional[Sequence[int]] = None) -> None:
    """One dynamic block.  Code lengths default to Huffman codes of the tokens' symbols; `dist_lens` may be all zero (an empty
    distance code) when the tokens hold no match."""
    lf, df = [0] * 286, [0] * 30
    for lit, dist in _symbols(tokens):
        if dist is None:
            lf[lit] += 1
        else:
            lf[lit[0]] += 1
            df[dist[0]] += 1
    lf[256] += 1
    lit_lens = list(lit_lens) if lit_lens is not None else huffman_lengths(lf)
    dist_lens = list(dist_lens) if dist_lens is not None else (huffman_lengths(df) if any(df) else [0])
    nlen = max(257, max(i for i, l in enumerate(lit_lens) if l) + 1)
    ndist = max(1, max((i for i, l in enumerate(dist_lens) if l), default=0) + 1)
    lens = lit_lens[:nlen] + (dist_lens + [0] * 30)[:ndist]
    cl = cl_lens if cl_lens is not None else huffman_lengths([lens.count(s) for s in range(19)], 7)
    cl_codes = canonical(cl)
    ncode = max(4, max(i for i, s in enumerate(CL_ORDER) if cl[s]) + 1)
    w.bits(int(final), 1)
    w.bits(2, 2)
    w.bits(nlen - 257, 5)
    w.bits(ndist - 1, 5)
    w.bits(ncode - 4, 4)
    for i in range(ncode):
        w.bits(cl[CL_ORDER[i]], 3)
    for l in lens:
        w.code(cl_codes[l], cl[l])
    _write_tokens(w, tokens, canonical(lit_lens), lit_lens, canonical((dist_lens + [0] * 30)[:30]), (dist_lens + [0] * 30)[:30])


def dynamic_header(w: BitWriter, final: bool, nlen: int, ndist: int, cl_lens: Sequence[int], lengths: Sequence,
                   ncode: int = 19) -> None:
    """A dynamic block header as written, checked by nothing: HLIT = nlen - 257 and HDIST = ndist - 1 (5 bits each, so 287 /
    288 and 31 / 32 are allowed), the first `ncode` of `cl_lens` (indexed by code-length symbol) in CL_ORDER, then `lengths`
    coded with the code of `cl_lens`: a length 0..15, a repeat (16 | 17 | 18, extra bits), or ("raw", value, bits)."""
    w.bits(int(final), 1)
    w.bits(2, 2)
    w.bits(nlen - 257, 5)
    w.bits(ndist - 1, 5)
    w.bits(ncode - 4, 4)
    for i in range(ncode):
        w.bits(cl_lens[CL_ORDER[i]], 3)
    codes = canonical(cl_lens)
    nbits = {16: 2, 17: 3, 18: 7}
    for x in lengths:
        if isinstance(x, tuple) and x[0] == "raw":
            w.bits(x[1], x[2])
        elif isinstance(x, tuple):
            w.code(codes[x[0]], cl_lens[x[0]])
            w.bits(x[1], nbits[x[0]])
        else:
            w.code(codes[x], cl_lens[x])


def tokens_with(w: BitWriter, tokens: Sequence[Token], lit_lens: Sequence[int], dist_lens: Sequence[int]) -> None:
    """The tokens and the end-of-block code, with explicit literal/length and distance code lengths (behind ``dynamic_header``)."""
    dist_lens = (list(dist_lens) + [0] * 30)[:30]
    _write_tokens(w, tokens, canonical(lit_lens), lit_lens, canonical(dist_lens), dist_lens)


def zlib_wrap(deflate: bytes, data: bytes) -> bytes:
    """The zlib stream of a raw DEFLATE stream that inflates to `data`: header 78 01, the blocks, Adler-32 of `data`."""
    return b"\x78\x01" + deflate + zlib.adler32(data).to_bytes(4, "big")


def expand(tokens: Sequence[Token], history: bytes = b"") -> bytes:
    """What the tokens inflate to after `history`."""
    out = bytearray(history)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            length, dist = t[0], t[1]
            for _ in range(length):
                out.append(out[-dist])
    return bytes(out[len(history):])
