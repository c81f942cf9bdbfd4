"""What PIL gives for a PNG's zlib stream, and what the GPU inflate's status words must say about it.  Plain Python, no GPU.

``inflate_as_pil(png)`` is a serial RFC 1950/1951 inflate with zlib's error rules, fed the way Pillow feeds it:
``ImageFile.load`` reads at most 64 KiB at a time and ``PngImageFile.load_read`` never crosses an IDAT (empty IDATs give no
read); ``ZipDecode.c`` calls ``inflate`` while the read has input, with room for the rest of one row, and stops after the call
that completes the last row, or after a call that completes a row and returns Z_STREAM_END.  zlib takes input a byte at a time
only when it needs more bits, decodes the next symbol even when it has no room to write it, and checks a distance against its
window only when it has room to copy.  So after the image's last byte zlib checks only what is left of the read that completed
it, and an image left short decodes only when the call that filled its last row also read the final Adler-32.

``chunk_status(stream, raw_len)`` restates csrc/png.cu's speculative chunk search (strict_header / strict_dynamic), its chunk
decode and the chain that links the chunks from the stream's start, and gives the status words [1..3] the decode must report:
chunks, chunks after the first whose start the chain confirmed, and the longest chunk's output when the chain decoded the
image (else the bytes the serial decoder wrote).
"""
from __future__ import annotations

import struct
import zlib
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from oracle.deflate_ref import DBASE, DEXT, LBASE, LEXT, CL_ORDER, FIXED_LIT

PIL_READ = 65536            # ImageFile.MAXBLOCK
CHUNK_BYTES = 65536         # csrc/png.cu: compressed bytes per speculative chunk
MAX_CHUNKS = 4096
CHUNK_SYMBOLS = 4 * 65536 + 131072
WINDOW = 32768


class Refused(Exception):
    """PIL refuses the file (zlib's error, a truncated image or a bad filter type)."""


# ---------------------------------------------------------------------------------------------------------------------
# bits and codes

class _Bits:
    """LSB-first bits of `data` from bit `pos`; reads past the end see zeros, `has` tells whether they exist."""

    def __init__(self, data: bytes, pos: int = 0):
        self.buf = bytes(data) + bytes(16)
        self.total = 8 * len(data)
        self.pos = pos

    def has(self, n: int) -> bool:
        return self.pos + n <= self.total

    def peek(self, n: int) -> int:
        b = self.pos >> 3
        return (int.from_bytes(self.buf[b:b + 6], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def take(self, n: int) -> int:
        v = self.peek(n)
        self.pos += n
        return v

    def taken(self) -> int:
        """Bytes zlib has pulled in to read every bit up to here."""
        return (self.pos + 7) >> 3


class _Code:
    """A canonical Huffman code, decoded through a table of every pattern of its longest length.  zlib calls a pattern invalid
    once the bits read rule out every code: for the codes it lets through (complete, one code of one bit, or empty) that is
    after max(1, longest length) bits."""

    def __init__(self, lengths: Sequence[int]):
        count = [0] * 16
        for l in lengths:
            count[l] += 1
        count[0] = 0
        code, nxt = 0, [0] * 16
        for b in range(1, 16):
            code = (code + count[b - 1]) << 1
            nxt[b] = code
        self.bits = max([l for l in range(16) if count[l]] or [1])
        self.table: List[Optional[Tuple[int, int]]] = [None] * (1 << self.bits)
        for s, l in enumerate(lengths):
            if l:
                rev = int(format(nxt[l], f"0{l}b")[::-1], 2)
                nxt[l] += 1
                for f in range(rev, 1 << self.bits, 1 << l):
                    self.table[f] = (s, l)

    def decode(self, br: "_Bits") -> Optional[int]:
        """The symbol, -1 for an invalid code, None when the code needs bits past the end."""
        e = self.table[br.peek(self.bits)]
        s, l = (-1, self.bits) if e is None else e
        if not br.has(l):
            return None
        br.pos += l
        return s


def _kraft_left(lengths: Sequence[int]) -> int:
    """2^15 minus the code space the lengths use: 0 complete, > 0 incomplete, < 0 over-subscribed."""
    return (1 << 15) - sum(1 << (15 - l) for l in lengths if l)


FIXED_LIT_CODE = _Code(FIXED_LIT)
FIXED_DIST_CODE = _Code([5] * 32)


class _Bad(Exception):
    pass


class _More(Exception):
    pass


def _read_dynamic(br: _Bits):
    """zlib's dynamic header: (literal/length code, distance code).  Raises _Bad (with the bytes zlib has taken when it refuses)
    or _More (it would wait for input).  zlib's rules: HLIT <= 286, HDIST <= 30; the code-length code complete (all zero
    passes here, reads each length as a 0 of one bit and then lacks an end-of-block code); a repeat 16 needs a previous length,
    and zlib reads its two extra bits first; no repeat past HLIT + HDIST; an end-of-block code; literal/length and distance
    codes that are complete or one code of one bit; an empty distance code passes."""
    if not br.has(14):
        raise _More
    nlen, ndist, ncode = br.take(5) + 257, br.take(5) + 1, br.take(4) + 4
    if nlen > 286 or ndist > 30:
        raise _Bad
    cl = [0] * 19
    for i in range(ncode):
        if not br.has(3):
            raise _More
        cl[CL_ORDER[i]] = br.take(3)
    if any(cl):
        if _kraft_left(cl):
            raise _Bad
        clc = _Code(cl)
    else:
        if not br.has(nlen + ndist):
            raise _More
        br.pos += nlen + ndist
        raise _Bad
    lens: List[int] = []
    while len(lens) < nlen + ndist:
        s = clc.decode(br)
        if s is None:
            raise _More
        if s < 16:
            lens.append(s)
            continue
        nb, base = {16: (2, 3), 17: (3, 3), 18: (7, 11)}[s]
        if not br.has(nb):
            raise _More
        rep = base + br.take(nb)
        if s == 16 and not lens:
            raise _Bad
        val = lens[-1] if s == 16 else 0
        if len(lens) + rep > nlen + ndist:
            raise _Bad
        lens += [val] * rep
    lit, dist = lens[:nlen], lens[nlen:]
    if lit[256] == 0:
        raise _Bad
    for part, allow_empty in ((lit, False), (dist, True)):
        left = _kraft_left(part)
        longest = max(part)
        if left < 0 or (left > 0 and longest != 1 and not (allow_empty and longest == 0)):
            raise _Bad
    return _Code(lit), _Code(dist)


# ---------------------------------------------------------------------------------------------------------------------
# the serial inflate as a list of events

def _events(z: bytes, total: int):
    """zlib's inflate of the whole stream `z`, as events in order, each with the bytes zlib has taken in at that point:
    ("w", taken, bytes, bad)  a literal or match to write (bad: its distance reaches before the output);
    ("s", taken, byte)        one stored byte (taken counts the byte itself);
    ("x", taken)              an error;
    ("e", taken)              the Adler-32 read and good: Z_STREAM_END;
    ("m", len(z) + 1)         the stream ended where zlib wants more.
    Stops after the first write the image has no room for (zlib would wait there for room PIL never gives)."""
    ev = []
    o = 0
    out = bytearray()
    if len(z) < 2:
        return [("m", len(z) + 1)]
    cmf, flg = z[0], z[1]
    if (cmf & 15) != 8 or (cmf >> 4) > 7 or (cmf << 8 | flg) % 31 or flg & 0x20:
        return [("x", 2)]
    br = _Bits(z, 16)
    last = False
    try:
        while True:
            if last:
                br.pos = (br.pos + 7) & ~7
                if not br.has(32):
                    raise _More
                v = br.take(32)
                v = int.from_bytes(v.to_bytes(4, "little"), "big")
                ev.append(("e", br.taken()) if v == zlib.adler32(bytes(out)) else ("x", br.taken()))
                return ev
            if not br.has(3):
                raise _More
            last = bool(br.take(1))
            kind = br.take(2)
            if kind == 3:
                raise _Bad
            if kind == 0:
                br.pos = (br.pos + 7) & ~7
                if not br.has(32):
                    raise _More
                ln, nln = br.take(16), br.take(16)
                if ln != nln ^ 0xFFFF:
                    raise _Bad
                for _ in range(ln):
                    if not br.has(8):
                        raise _More
                    b = br.take(8)
                    ev.append(("s", br.taken(), b))
                    if o >= total:
                        return ev
                    out.append(b)
                    o += 1
                continue
            lit, dist = (FIXED_LIT_CODE, FIXED_DIST_CODE) if kind == 1 else _read_dynamic(br)
            while True:
                s = lit.decode(br)
                if s is None:
                    raise _More
                if s < 0 or s > 285:
                    raise _Bad
                if s < 256:
                    ev.append(("w", br.taken(), bytes([s]), False))
                    if o >= total:
                        return ev
                    out.append(s)
                    o += 1
                    continue
                if s == 256:
                    break
                if not br.has(LEXT[s - 257]):
                    raise _More
                length = LBASE[s - 257] + br.take(LEXT[s - 257])
                ds = dist.decode(br)
                if ds is None:
                    raise _More
                if ds < 0 or ds > 29:
                    raise _Bad
                if not br.has(DEXT[ds]):
                    raise _More
                d = DBASE[ds] + br.take(DEXT[ds])
                if o >= total or d > o:
                    ev.append(("w", br.taken(), None, True))
                    return ev
                n = min(length, total - o)
                for _ in range(n):
                    out.append(out[-d])
                ev.append(("w", br.taken(), bytes(out[o:o + n]) + bytes(length - n), False))
                o += n
                if n < length:
                    return ev
    except _Bad:
        ev.append(("x", br.taken()))
    except _More:
        ev.append(("m", len(z) + 1))
    return ev


# ---------------------------------------------------------------------------------------------------------------------
# PNG files as PIL reads them

def png_parts(png: bytes):
    """(IHDR fields (w, h, color, depth, interlace), PLTE bytes or None, IDAT payloads) of a PNG file, chunk CRCs unchecked."""
    pos, hdr, plte, idat = 8, None, None, []
    while pos + 8 <= len(png):
        n = struct.unpack(">I", png[pos:pos + 4])[0]
        kind, data = png[pos + 4:pos + 8], png[pos + 8:pos + 8 + n]
        if kind == b"IHDR":
            w, h, depth, color, _, _, interlace = struct.unpack(">IIBBBBB", data)
            hdr = (w, h, color, depth, interlace)
        elif kind == b"PLTE":
            plte = data
        elif kind == b"IDAT":
            idat.append(data)
        elif kind == b"IEND":
            break
        pos += 12 + n
    return hdr, plte, idat


def row_bytes(w: int, color: int, depth: int) -> int:
    return (w * {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[color] * depth + 7) // 8


def pil_reads(idat: Sequence[bytes]) -> List[int]:
    """The end offsets in the zlib stream of the reads Pillow hands zlib: each non-empty IDAT in 64 KiB pieces from its start."""
    ends, at = [], 0
    for d in idat:
        for k in range(0, len(d), PIL_READ):
            ends.append(at + min(len(d), k + PIL_READ))
        at += len(d)
    return ends


def feed_as_pil(ev, reads: Sequence[int], total: int, row: int) -> Union[int, Refused]:
    """Drives zlib (its events `ev` from ``_events``) as Pillow does (`reads`: their end offsets): how many filtered bytes PIL
    keeps, or why it refuses."""
    r, end = 0, reads[0]
    o = 0
    full = False        # the current call filled a row that PIL has not taken yet

    def next_read():
        nonlocal r, end
        r += 1
        if r == len(reads):
            raise Refused("image file is truncated")
        end = reads[r]

    try:
        for e in ev:
            kind, need = e[0], e[1]
            if need > end:              # the call runs out of input first: PIL takes a filled row, then reads on
                if full:
                    full = False
                    if o >= total:
                        return o
                while need > end:
                    next_read()
            if kind == "x":
                raise Refused("broken data stream")
            if kind == "e":
                if full:                # Z_STREAM_END in the call that filled a row
                    return o
                raise Refused("image file is truncated")
            if kind == "m":
                raise Refused("image file is truncated")
            taken = need - 1 if kind == "s" else need       # a stored byte is taken as it is written
            n = 1 if kind == "s" else len(e[2]) if e[2] is not None else 1
            if full:                    # no room: zlib returns, PIL takes the row and calls again
                full = False
                if o >= total:
                    return o
                if taken == end:
                    next_read()
            if kind == "w" and e[3]:
                raise Refused("invalid distance too far back")
            while n:
                k = min(n, row - o % row)
                o += k
                n -= k
                if o % row == 0:
                    if not n:
                        full = True
                        break
                    if o >= total:      # a match past the image's end
                        return o
                    if taken == end:
                        next_read()
        raise AssertionError("events end without a verdict")
    except Refused as e:
        return e


def inflate_as_pil(png: bytes) -> Union[bytes, Refused]:
    """The filtered rows PIL decodes from a non-interlaced PNG (fewer than the image's when the stream ends cleanly on a row
    boundary), or ``Refused``."""
    (w, h, color, depth, interlace), _, idat = png_parts(png)
    assert not interlace
    row = 1 + row_bytes(w, color, depth)
    z = b"".join(idat)
    reads = pil_reads(idat)
    if not reads:
        return Refused("image file is truncated")
    ev = _events(z, h * row)
    got = feed_as_pil(ev, reads, h * row, row)
    if isinstance(got, Refused):
        return got
    raw = _events_bytes(ev, got)
    for r in range(0, got, row):
        if raw[r] > 4:
            return Refused("unrecognized filter type")
    return raw


def _events_bytes(ev, n: int) -> bytes:
    out = bytearray()
    for e in ev:
        if e[0] == "s":
            out.append(e[2])
        elif e[0] == "w" and e[2] is not None:
            out += e[2]
    return bytes(out[:n])


def serial_bytes(z: bytes, total: int) -> int:
    """The bytes csrc/png.cu's serial decoder writes from the whole stream before it stops (its status word 3)."""
    o = 0
    for e in _events(z, total):
        if e[0] == "s" or (e[0] == "w" and not e[3]):
            o = min(total, o + (1 if e[0] == "s" else len(e[2])))
    return o


def unfilter(raw: bytes, w: int, h: int, color: int, depth: int) -> np.ndarray:
    """The unfiltered rows, uint8 [h, rowbytes], of filtered rows `raw` (rows it lacks are zero, as in PIL's image)."""
    rb = row_bytes(w, color, depth)
    bpp = max(1, {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[color] * depth // 8)
    out = np.zeros((h, rb), np.int64)
    prev = np.zeros(rb, np.int64)
    for r in range(len(raw) // (rb + 1)):
        f, cur = raw[r * (rb + 1)], np.frombuffer(raw, np.uint8, rb, r * (rb + 1) + 1).astype(np.int64)
        rec = np.zeros(rb, np.int64)
        for x in range(rb):
            a = rec[x - bpp] if x >= bpp else 0
            b = prev[x]
            c = prev[x - bpp] if x >= bpp else 0
            if f == 0:
                p = 0
            elif f == 1:
                p = a
            elif f == 2:
                p = b
            elif f == 3:
                p = (a + b) >> 1
            else:
                pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                p = a if pa <= pb and pa <= pc else b if pb <= pc else c
            rec[x] = (cur[x] + p) & 255
        out[r] = rec
        prev = rec
    return out.astype(np.uint8)


def pixels_as_pil(png: bytes) -> Union[np.ndarray, Refused]:
    """``read_image`` of an 8-bit grey, RGB, grey + alpha or RGBA PNG, from ``inflate_as_pil``: uint8 [h, w, 3] or ``Refused``."""
    (w, h, color, depth, _), _, _ = png_parts(png)
    assert depth == 8 and color in (0, 2, 4, 6)
    raw = inflate_as_pil(png)
    if isinstance(raw, Refused):
        return raw
    ch = {0: 1, 2: 3, 4: 2, 6: 4}[color]
    px = unfilter(raw, w, h, color, depth).reshape(h, w, ch)
    return np.repeat(px[..., :1], 3, axis=2) if ch < 3 else px[..., :3].copy()


# ---------------------------------------------------------------------------------------------------------------------
# the chunk-parallel path's status words

def _strict_dynamic(br: _Bits) -> bool:
    if not br.has(14):
        return False
    nlen, ndist, ncode = br.take(5) + 257, br.take(5) + 1, br.take(4) + 4
    if nlen > 286 or ndist > 30 or not br.has(3 * ncode):
        return False
    cl = [0] * 19
    for i in range(ncode):
        cl[CL_ORDER[i]] = br.take(3)
    if not any(cl) or _kraft_left(cl):
        return False
    clc = _Code(cl)
    lens: List[int] = []
    while len(lens) < nlen + ndist:
        s = clc.decode(br)
        if s is None or s < 0:
            return False
        if s < 16:
            lens.append(s)
            continue
        nb, base = {16: (2, 3), 17: (3, 3), 18: (7, 11)}[s]
        if (s == 16 and not lens) or not br.has(nb):
            return False
        rep = base + br.take(nb)
        if len(lens) + rep > nlen + ndist:
            return False
        lens += [lens[-1] if s == 16 else 0] * rep
    lit, dist = lens[:nlen], lens[nlen:]
    if not lit[256]:
        return False
    ll, dl = _kraft_left(lit), _kraft_left(dist)
    return ll >= 0 and dl >= 0 and (ll == 0 or max(lit) == 1) and (dl == 0 or max(dist) <= 1)


def _stored_len(br: _Bits) -> int:
    pad = (8 - (br.pos & 7)) & 7
    if br.take(pad):
        return -1
    if not br.has(32):
        return -1
    ln, nln = br.take(16), br.take(16)
    return ln if ln == nln ^ 0xFFFF else -1


def strict_header(stream: bytes, bit: int, br: Optional[_Bits] = None) -> bool:
    """csrc/png.cu strict_header: a block header at `bit` that parses strictly (a dynamic header by zlib's rules, or a stored
    header with zero padding, LEN == ~NLEN and a header that parses behind its data)."""
    br = br or _Bits(stream)
    br.pos = bit
    if not br.has(3):
        return False
    kind = br.take(3) >> 1
    if kind == 2:
        return _strict_dynamic(br)
    if kind != 0:
        return False
    ln = _stored_len(br)
    if ln < 0:
        return False
    after = br.pos + 8 * ln
    if after + 3 > br.total:
        return True
    br.pos = after
    kind = br.take(3) >> 1
    if kind == 0:
        return _stored_len(br) >= 0
    if kind == 2:
        return _strict_dynamic(br)
    return kind == 1


def _field(bits: np.ndarray, at: np.ndarray, n: int) -> np.ndarray:
    v = np.zeros(at.shape, np.int64)
    for i in range(n):
        v |= bits[at + i].astype(np.int64) << i
    return v


def find_candidate(stream: bytes, b0: int, b1: int) -> int:
    """The first bit in [b0, b1) where ``strict_header`` holds, or -1 (png_find_kernel).  Positions that cannot pass (block
    type, field limits, an incomplete code-length code, stored padding or LEN / NLEN) are ruled out in bulk first."""
    total = 8 * len(stream)
    buf = np.frombuffer(bytes(stream) + bytes(16), np.uint8)
    bits = np.unpackbits(buf, bitorder="little")
    buf = buf.astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(bits, dtype=np.int64)])
    br = _Bits(stream)
    for s0 in range(b0, b1, 8192):
        p = np.arange(s0, min(b1, s0 + 8192), dtype=np.int64)
        for q in p[_may_parse(bits, buf, cs, p, total)]:
            if strict_header(stream, int(q), br):
                return int(q)
    return -1


def _may_parse(bits, buf, cs, p, total):
    kind = _field(bits, p + 1, 2)
    ok = np.zeros(p.shape, bool)
    # dynamic: HLIT, HDIST, and a complete code-length code
    dyn = (kind == 2) & (p + 17 <= total) & (_field(bits, p + 3, 5) <= 29) & (_field(bits, p + 8, 5) <= 29)
    ncode = _field(bits, p + 13, 4) + 4
    dyn &= p + 17 + 3 * ncode <= total
    kraft = np.zeros(p.shape, np.int64)
    for i in range(19):
        l = _field(bits, p + 17 + 3 * i, 3)
        kraft += np.where((i < ncode) & (l > 0), 1 << (7 - l), 0)
    ok |= dyn & (kraft == 128)
    # stored: zero padding, LEN == ~NLEN
    a = (p + 3 + 7) & ~7
    st = (kind == 0) & (p + 3 <= total) & (cs[a] - cs[p + 3] == 0) & (a + 32 <= total)
    byte = a >> 3
    b = buf
    ln = b[byte] | b[byte + 1] << 8
    nln = b[byte + 2] | b[byte + 3] << 8
    return ok | (st & ((ln ^ nln) == 0xFFFF))


def plan_chunks(stream_len: int) -> Tuple[int, int]:
    """(chunk bytes, chunks) as k2y_png_plan cuts a stream."""
    cb = max(CHUNK_BYTES, -(-stream_len // MAX_CHUNKS))
    return cb, max(1, -(-stream_len // cb))


def candidates(stream: bytes) -> List[int]:
    cb, n = plan_chunks(len(stream))
    return [16] + [find_candidate(stream, k * cb * 8, min(8 * len(stream), (k + 1) * cb * 8)) for k in range(1, n)]


def chunk_status(stream: bytes, raw_len: int, cands: Optional[List[int]] = None) -> List[int]:
    """Status words [1..3] of the GPU decode of zlib stream `stream` into `raw_len` filtered bytes: chunks; chunks after the first
    the chain from the stream's start confirmed (each chunk decodes from its candidate until it stands on a later chunk's
    candidate at a block boundary, ends the final block, or fails: invalid data, a distance before its 32 KiB window, more output
    than its capacity, the stream's end); and, when the chain ends the final block after exactly `raw_len` bytes with a good
    Adler-32 behind it, the longest chunk's output, else the bytes the serial decoder writes."""
    cands = candidates(stream) if cands is None else cands
    n = len(cands)
    br = _Bits(stream, 16)
    out = bytearray()
    chain, lens = [0], [0]
    cur, o, fails, bad_ref, final = 0, 0, False, False, False
    cap = raw_len

    def link():
        j = next((k for k in range(cur + 1, n) if cands[k] >= 0 and cands[k] >= br.pos), n)
        return j if j < n and cands[j] == br.pos else -1

    try:
        while True:
            j = link()
            if j >= 0:
                chain.append(j)
                lens.append(0)
                cur, o, cap = j, 0, min(raw_len, CHUNK_SYMBOLS)
            if not br.has(3):
                raise _Bad
            last = br.take(1)
            kind = br.take(2)
            if kind == 3:
                raise _Bad
            if kind == 0:
                br.pos = (br.pos + 7) & ~7
                if not br.has(32):
                    raise _Bad
                ln, nln = br.take(16), br.take(16)
                if ln != nln ^ 0xFFFF or o + ln > cap or not br.has(8 * ln):
                    raise _Bad
                out += bytes(br.take(8) for _ in range(ln))
                o += ln
            else:
                try:
                    lit, dist = (FIXED_LIT_CODE, FIXED_DIST_CODE) if kind == 1 else _read_dynamic(br)
                except _More:
                    raise _Bad
                while True:
                    s = lit.decode(br)
                    if s is None or s < 0 or s > 285:
                        raise _Bad
                    if s < 256:
                        if o >= cap:
                            raise _Bad
                        out.append(s)
                        o += 1
                        continue
                    if s == 256:
                        break
                    if not br.has(LEXT[s - 257]):
                        raise _Bad
                    length = LBASE[s - 257] + br.take(LEXT[s - 257])
                    ds = dist.decode(br)
                    if ds is None or ds < 0 or ds > 29 or not br.has(DEXT[ds]):
                        raise _Bad
                    d = DBASE[ds] + br.take(DEXT[ds])
                    if d > o + (WINDOW if cur else 0) or o + length > cap:
                        raise _Bad
                    for _ in range(length):
                        if len(out) - d < 0:
                            bad_ref = True
                            out.append(0)
                        else:
                            out.append(out[-d])
                    o += length
            lens[-1] = o
            if last:
                final = True
                break
    except _Bad:
        fails = True
    if fails:                   # the failing chunk is not part of the chain
        chain.pop()
        lens.pop()
    confirmed = max(0, len(chain) - 1)
    good = final and not fails and len(out) == raw_len and not bad_ref
    if good:
        at = (br.pos + 7) >> 3
        good = at + 4 <= len(stream) and stream[at:at + 4] == zlib.adler32(bytes(out)).to_bytes(4, "big")
    return [n, confirmed, max(lens) if good else serial_bytes(stream, raw_len)]
