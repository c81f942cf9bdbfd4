"""TEST INFRASTRUCTURE — a sequential-Huffman JPEG writer with every knob explicit, and an exact integer decoder back end.

Only tests/ may import this module; the product path is k210_yolo_framework_b200/csrc/jpeg.cu.

Writer (`write_jpeg`): quantised coefficients in, file bytes out.  The caller picks SOF0 / SOF1, component ids, frame and
scan order, sampling factors, 8- or 16-bit quantisation tables with ids 0-3, Huffman tables (the standard ones of ITU T.81
Annex K.3, optimal ones built from the data with libjpeg's jpeg_gen_optimal_table, or any hand-made code-length
distribution) with ids 0-3, the restart interval (and an extra RSTn after the last interval), the pad bits (ones, zeros,
random), runs of 0xFF fill bytes before markers, extra APPn / COM segments, and where DQT / DHT go (before the frame header,
after it, or defined once with other content and redefined before the scan).  It reports each restart segment's length in
bits, before padding, so tests can place segment ends and codewords on chosen bit positions.

`pixels_to_coefs` turns an RGB or grey image into conforming coefficients (level shift, float64 DCT, rounding quantisation,
box-filtered chroma for subsampled layouts).

Decoder back end (`decode_coefs`): what a decoder does after the Huffman stage, as PIL runs it on x86-64: dequantisation and
libjpeg-turbo's x86 SIMD `islow` IDCT (jidctint-avx2.asm / jidctint-sse2.asm: 16-bit dequantised products, 16-bit sums
feeding the multiplies, 32-bit multiply-accumulate, pass-1 results packed to int16 with saturation, pass-2 results packed
to int16 and then int8 with saturation; and, when rows 1-7 of the whole block are zero, a pass 1 that shifts the 16-bit row 0
left by two bits without saturating), libjpeg-turbo's upsampler dispatch with fancy upsampling on (jinit_upsampler,
including the box filters it picks when the downsampled width is at most 2) and ycc_rgb_convert.  This differs from
jidctint.c (libjpeg-turbo's C path, 32-bit throughout with a masked range-limit table) once dequantised coefficients leave
the range a conforming 8-bit encoder writes.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# natural (row-major) index of zig-zag position k
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63])

# Luma sampling factors by layout; chroma is 1x1.  "gray" is one component.
LAYOUTS = {"444": (1, 1), "422": (2, 1), "440": (1, 2), "420": (2, 2), "411": (4, 1), "gray": (1, 1)}

# ITU T.81 Annex K.3 (bits[1..16], values)
STD_DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
STD_DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
STD_AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16,
    0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6,
    0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8,
    0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
STD_AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34,
    0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4,
    0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6,
    0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])

# ITU T.81 Annex K.1, natural order
STD_Q_LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22,
                       29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87,
                       103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
STD_Q_CHROMA = np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66,
                         99, 99, 99, 99, 99, 99] + [99] * 32)


def quality_table(base: np.ndarray, quality: int) -> np.ndarray:
    """libjpeg's jpeg_quality_scaling of a base table, clamped to 1..255."""
    s = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * s + 50) // 100, 1, 255)


# ---------------------------------------------------------------------------------------------------------------------
# Huffman tables
# ---------------------------------------------------------------------------------------------------------------------
def table_from_lengths(lengths: Dict[int, int]) -> Tuple[List[int], List[int]]:
    """(bits[1..16], values) of a canonical table giving each symbol its code length (symbols of one length by value)."""
    assert lengths and all(1 <= l <= 16 for l in lengths.values())
    # libjpeg refuses a table whose codes of some length end in the all-ones code: keep the Kraft sum below 1
    assert sum(2.0 ** -l for l in lengths.values()) < 1.0, "code lengths leave no room for the reserved all-ones code"
    bits = [0] * 16
    vals = []
    for l in range(1, 17):
        syms = sorted(s for s, n in lengths.items() if n == l)
        bits[l - 1] = len(syms)
        vals += syms
    return bits, vals


def optimal_table(freq: Dict[int, int]) -> Tuple[List[int], List[int]]:
    """libjpeg's jpeg_gen_optimal_table (jchuff.c): Huffman code lengths limited to 16 bits, the all-ones code reserved."""
    f = np.zeros(257, np.int64)
    for s, n in freq.items():
        f[s] = n
    f[256] = 1
    codesize = np.zeros(257, np.int64)
    others = np.full(257, -1, np.int64)
    while True:
        c1, v = -1, 1 << 62
        for i in range(257):
            if 0 < f[i] <= v:
                v, c1 = f[i], i
        c2, v = -1, 1 << 62
        for i in range(257):
            if 0 < f[i] <= v and i != c1:
                v, c2 = f[i], i
        if c2 < 0:
            break
        f[c1] += f[c2]
        f[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = np.zeros(33, np.int64)
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1   # the reserved code
    vals = [j for l in range(1, 33) for j in range(256) if codesize[j] == l]
    return [int(b) for b in bits[1:17]], vals


def flat_table(symbols: Sequence[int], length: int) -> Tuple[List[int], List[int]]:
    """Every symbol at one code length."""
    return table_from_lengths({s: length for s in symbols})


def _codes(spec) -> Dict[int, Tuple[int, int]]:
    bits, vals = spec
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


def _category(v: int) -> int:
    return int(abs(int(v))).bit_length()


def _magnitude_bits(v: int, s: int) -> int:
    return v if v >= 0 else v + (1 << s) - 1


# ---------------------------------------------------------------------------------------------------------------------
# Writer
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Written:
    data: bytes
    seg_bits: List[int]        # codeword bits of each restart segment, before padding
    coefs: List[np.ndarray]    # per frame component [bh, bw, 8, 8] natural order, DC as the decoder stores it (int16)
    qt: List[np.ndarray]       # per frame component, natural order, as latched at the scan
    sampling: List[Tuple[int, int]]
    height: int
    width: int


def block_grid(height: int, width: int, sampling: Sequence[Tuple[int, int]]) -> List[Tuple[int, int]]:
    """Blocks (rows, cols) of each component's coefficient array: MCU-padded, or one block per MCU for a grey frame."""
    if len(sampling) == 1:
        return [(-(-height // 8), -(-width // 8))]
    hmax = max(h for h, _ in sampling)
    vmax = max(v for _, v in sampling)
    mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    return [(my * v, mx * h) for h, v in sampling]


def _segment(marker: int, payload: bytes) -> bytes:
    assert len(payload) + 2 < 65536
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def _dqt(tables: Dict[int, np.ndarray], prec: Dict[int, int]) -> bytes:
    out = b""
    for tid, q in tables.items():
        q = np.asarray(q).reshape(64)
        p = prec[tid]
        out += bytes([(p << 4) | tid])
        for k in range(64):
            v = int(q[ZIGZAG[k]])
            out += v.to_bytes(2, "big") if p else bytes([v])
    return out


def _dht(tables: Dict[Tuple[str, int], Tuple[List[int], List[int]]]) -> bytes:
    out = b""
    for (cls, tid), (bits, vals) in tables.items():
        out += bytes([(1 if cls == "ac" else 0) << 4 | tid]) + bytes(bits) + bytes(vals)
    return out


def _bit_array(words: np.ndarray, lengths: np.ndarray) -> np.ndarray:
    """MSB-first bits of each (word, length <= 32), concatenated."""
    ends = np.cumsum(lengths)
    out = np.zeros(int(ends[-1]) if len(ends) else 0, np.uint8)
    starts = ends - lengths
    for j in range(32):
        m = lengths > j
        out[starts[m] + j] = (words[m] >> (lengths[m] - 1 - j)) & 1
    return out


def _stuff(bits: np.ndarray) -> bytes:
    assert len(bits) % 8 == 0
    return np.packbits(bits).tobytes().replace(b"\xff", b"\xff\x00")


def write_jpeg(coefs: Sequence[np.ndarray], qtables: Dict[int, np.ndarray], *, height: int, width: int,
               sampling: Sequence[Tuple[int, int]], tq: Optional[Sequence[int]] = None, qprec: Optional[Dict[int, int]] = None,
               ids: Optional[Sequence[int]] = None, scan_order: Optional[Sequence[int]] = None, sof: int = 0xC0,
               huffman="std", hsel: Optional[Sequence[Tuple[int, int]]] = None, restart: int = 0, extra_rst: bool = False,
               pad: str = "ones", tail_bytes: int = 0, fill: int = 0, segments: Sequence[Tuple[int, bytes]] = (),
               tables: str = "before_sof", jfif: bool = True, seed: int = 0) -> Written:
    """One baseline / extended sequential Huffman JPEG, one scan with every component.

    coefs      per frame component, int [bh, bw, 8, 8] in natural order at `block_grid` size; DC as absolute values, written
               as differences modulo 2^16 (the decoder's running sum may pass +-32767; it stores the low 16 bits)
    qtables    table id (0-3) -> 64 values in natural order; `tq` picks one per component (default 0 for the first, 1 for the
               others, or 0 when only table 0 is given); `qprec` id -> 0 (8-bit) / 1 (16-bit), default 16-bit where a value
               exceeds 255
    ids        component ids in frame order; `scan_order`: frame indices in the order the scan lists them (and the MCU
               holds them)
    huffman    "std", "optimal", or a dict (cls "dc" / "ac", id) -> (bits, values) | "std" | "optimal"; `hsel`: (DC id, AC id)
               per frame component (default (0, 0) for the first, (1, 1) for the others)
    restart    DRI interval in MCUs (0: none); `extra_rst` writes one more RSTn after the last interval
    pad        "ones", "zeros" or "random" bits to the byte boundary at each segment end, then `tail_bytes` whole bytes of them
    fill       0xFF fill bytes before every RSTn and the EOI marker
    segments   (marker, payload) written after SOI (and APP0 when `jfif`)
    tables     "before_sof", "after_sof" (one DQT / DHT segment per table), or "redefined" (other content under the same ids
               before SOF, the real tables after it)
    """
    n = len(coefs)
    sampling = [tuple(s) for s in sampling]
    assert len(sampling) == n and n in (1, 3)
    ids = list(ids) if ids is not None else list(range(1, n + 1))
    scan_order = list(scan_order) if scan_order is not None else list(range(n))
    tq = list(tq) if tq is not None else [0 if c == 0 or len(qtables) == 1 else 1 for c in range(n)]
    hsel = list(hsel) if hsel is not None else [(0, 0) if c == 0 else (1, 1) for c in range(n)]
    qprec = dict(qprec) if qprec is not None else {t: int(np.max(q) > 255) for t, q in qtables.items()}
    grid = block_grid(height, width, sampling)
    coefs = [np.asarray(c, np.int64).reshape(gh, gw, 8, 8) for c, (gh, gw) in zip(coefs, grid)]
    rng = np.random.default_rng(seed)

    # MCU structure
    if n == 1:
        per_mcu = [[(0, by, bx)] for by in range(grid[0][0]) for bx in range(grid[0][1])]
    else:
        hmax = max(h for h, _ in sampling)
        vmax = max(v for _, v in sampling)
        mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
        per_mcu = []
        for m in range(mx * my):
            x, y = m % mx, m // mx
            per_mcu.append([(c, y * sampling[c][1] + j, x * sampling[c][0] + i) for c in scan_order
                            for j in range(sampling[c][1]) for i in range(sampling[c][0])])
    # symbols of each MCU: (component, class, symbol, extra value, extra bits)
    last = [0] * n
    stored = [c.copy() for c in coefs]
    seg_syms: List[List[Tuple[int, str, int, int, int]]] = []
    cur: List[Tuple[int, str, int, int, int]] = []
    for m, blocks in enumerate(per_mcu):
        if restart and m and m % restart == 0:
            seg_syms.append(cur)
            cur = []
            last = [0] * n
        for c, by, bx in blocks:
            blk = coefs[c][by, bx].reshape(64)
            dc = int(blk[0])
            d = ((dc - last[c] + 32768) & 0xFFFF) - 32768
            if d == -32768:
                raise ValueError(f"DC difference of -32768 (component {c}, block {by},{bx}) has no code")
            last[c] += d
            stored[c][by, bx, 0, 0] = ((last[c] + 32768) & 0xFFFF) - 32768
            s = _category(d)
            cur.append((c, "dc", s, _magnitude_bits(d, s), s))
            zz = blk[ZIGZAG]
            assert np.all(np.abs(zz[1:]) <= 32767), "AC coefficients beyond +-32767 have no code"
            run = 0
            nz = np.nonzero(zz[1:])[0]
            end = nz[-1] + 1 if len(nz) else 0
            for k in range(1, end + 1):
                v = int(zz[k])
                if v == 0:
                    run += 1
                    continue
                while run > 15:
                    cur.append((c, "ac", 0xF0, 0, 0))
                    run -= 16
                s = _category(v)
                assert s <= 15, "AC magnitude category above 15"
                cur.append((c, "ac", (run << 4) | s, _magnitude_bits(v, s), s))
                run = 0
            if end < 63:
                cur.append((c, "ac", 0x00, 0, 0))
    seg_syms.append(cur)

    # Huffman tables
    used = {("dc", hsel[c][0]) for c in range(n)} | {("ac", hsel[c][1]) for c in range(n)}
    spec = huffman if isinstance(huffman, dict) else {k: huffman for k in used}
    freq: Dict[Tuple[str, int], Dict[int, int]] = {k: {} for k in used}
    for seg in seg_syms:
        for c, cls, sym, _, _ in seg:
            key = (cls, hsel[c][0] if cls == "dc" else hsel[c][1])
            freq[key][sym] = freq[key].get(sym, 0) + 1
    htabs = {}
    for key in sorted(used):
        s = spec[key]
        if s == "std":
            s = (STD_DC_LUMA if key[1] == 0 else STD_DC_CHROMA) if key[0] == "dc" else (STD_AC_LUMA if key[1] == 0 else STD_AC_CHROMA)
        elif s == "optimal":
            s = optimal_table(freq[key])
        htabs[key] = (list(s[0]), list(s[1]))
    codes = {k: _codes(v) for k, v in htabs.items()}

    # entropy-coded segments
    entropy = b""
    seg_bits = []
    for si, seg in enumerate(seg_syms):
        words, lens = np.zeros(len(seg), np.int64), np.zeros(len(seg), np.int64)
        for k, (c, cls, sym, val, nb) in enumerate(seg):
            table = codes[(cls, hsel[c][0] if cls == "dc" else hsel[c][1])]
            if sym not in table:
                raise ValueError(f"symbol 0x{sym:02X} is not in the {cls} table of component {c}")
            code, l = table[sym]
            words[k], lens[k] = (code << nb) | val, l + nb
        bits = _bit_array(words, lens)
        seg_bits.append(len(bits))
        npad = (-len(bits)) % 8 + 8 * tail_bytes
        padding = {"ones": np.ones(npad, np.uint8), "zeros": np.zeros(npad, np.uint8)}.get(pad)
        if padding is None:
            padding = rng.integers(0, 2, npad).astype(np.uint8)
        entropy += _stuff(np.concatenate([bits, padding]))
        if si + 1 < len(seg_syms) or extra_rst:
            entropy += b"\xff" * fill + bytes([0xFF, 0xD0 + si % 8])
    entropy += b"\xff" * fill + b"\xff\xd9"

    # headers
    sof_payload = bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([n])
    for c in range(n):
        sof_payload += bytes([ids[c], (sampling[c][0] << 4) | sampling[c][1], tq[c]])
    sos_payload = bytes([n])
    for c in scan_order:
        sos_payload += bytes([ids[c], (hsel[c][0] << 4) | hsel[c][1]])
    sos_payload += bytes([0, 63, 0])
    head = b"\xff\xd8"
    if jfif:
        head += _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for m, p in segments:
        head += _segment(m, p)
    qtables = {t: np.asarray(q, np.int64).reshape(64) for t, q in qtables.items()}
    if tables == "before_sof":
        head += _segment(0xDB, _dqt(qtables, qprec)) + _segment(0xC4, _dht(htabs)) + _segment(sof, sof_payload)
    elif tables == "after_sof":
        head += _segment(sof, sof_payload)
        for t in qtables:
            head += _segment(0xDB, _dqt({t: qtables[t]}, qprec))
        for k in htabs:
            head += _segment(0xC4, _dht({k: htabs[k]}))
    else:
        assert tables == "redefined"
        other_q = {t: np.full(64, 1 + t) for t in qtables}
        other_h = {k: flat_table(range(12) if k[0] == "dc" else range(255), 4 if k[0] == "dc" else 8) for k in htabs}
        head += _segment(0xDB, _dqt(other_q, {t: 0 for t in qtables})) + _segment(0xC4, _dht(other_h))
        head += _segment(sof, sof_payload) + _segment(0xDB, _dqt(qtables, qprec)) + _segment(0xC4, _dht(htabs))
    if restart:
        head += _segment(0xDD, restart.to_bytes(2, "big"))
    head += _segment(0xDA, sos_payload)
    return Written(head + entropy, seg_bits, stored, [qtables[tq[c]].copy() for c in range(n)], sampling, height, width)


# ---------------------------------------------------------------------------------------------------------------------
# Pixels -> conforming coefficients
# ---------------------------------------------------------------------------------------------------------------------
_DCT = np.array([[(np.sqrt(0.125) if u == 0 else 0.5) * np.cos((2 * x + 1) * u * np.pi / 16) for x in range(8)] for u in range(8)])


def _fdct_quant(plane: np.ndarray, q: np.ndarray) -> np.ndarray:
    gh, gw = plane.shape[0] // 8, plane.shape[1] // 8
    b = plane.reshape(gh, 8, gw, 8).transpose(0, 2, 1, 3) - 128.0
    d = np.einsum("ux,abxy,vy->abuv", _DCT, b, _DCT)
    return np.round(d / np.asarray(q, np.float64).reshape(8, 8)).astype(np.int64)


def pixels_to_coefs(img: np.ndarray, layout: str, qt: Sequence[np.ndarray]) -> Tuple[List[np.ndarray], List[Tuple[int, int]]]:
    """Conforming coefficients of an RGB (or, for "gray", grey) uint8 image: JFIF RGB->YCbCr in float64, edge-replicated
    to the block grid, chroma box-filtered for subsampled layouts, level shift, float64 DCT, rounding quantisation with
    qt[0] (luma) and qt[1] (chroma)."""
    h, w = img.shape[:2]
    hs, vs = LAYOUTS[layout]
    if layout == "gray":
        g = img.astype(np.float64) if img.ndim == 2 else img.astype(np.float64) @ np.array([0.299, 0.587, 0.114])
        (gh, gw), = block_grid(h, w, [(1, 1)])
        return [_fdct_quant(np.pad(g, ((0, gh * 8 - h), (0, gw * 8 - w)), mode="edge"), qt[0])], [(1, 1)]
    sampling = [(hs, vs), (1, 1), (1, 1)]
    grid = block_grid(h, w, sampling)
    x = img.astype(np.float64)
    y = x @ np.array([0.299, 0.587, 0.114])
    cb = x @ np.array([-0.168735892, -0.331264108, 0.5]) + 128
    cr = x @ np.array([0.5, -0.418687589, -0.081312411]) + 128
    ph, pw = grid[0][0] * 8, grid[0][1] * 8
    planes = [np.pad(p, ((0, ph - h), (0, pw - w)), mode="edge") for p in (y, cb, cr)]
    out = [_fdct_quant(planes[0], qt[0])]
    for p in planes[1:]:
        p = p.reshape(ph // vs, vs, pw // hs, hs).mean(axis=(1, 3))
        out.append(_fdct_quant(p, qt[1]))
    return out, sampling


def extreme_blocks(rng: np.random.Generator, n: int, kind: str) -> np.ndarray:
    """int64 [n, 8, 8] natural-order coefficients far outside what an 8-bit encoder writes.  "dc": DC anywhere in +-32767,
    rows 1-7 zero, row 0 AC nonzero in half the blocks; "full": 1-64 nonzero coefficients anywhere, from +-32767 down to +-1."""
    out = np.zeros((n, 64), np.int64)
    mag = lambda size: (rng.choice([1, 16, 256, 4096, 32768], size) * rng.random(size)).astype(np.int64) * rng.choice([-1, 1], size)
    if kind == "dc":
        out[:, 0] = rng.integers(-32767, 32768, n)
        row0 = rng.random(n) < 0.5
        out[row0, 1:8] = mag((int(row0.sum()), 7)) * (rng.random((int(row0.sum()), 7)) < 0.5)
    else:
        assert kind == "full"
        count = rng.integers(1, 65, n)
        keep = rng.random((n, 64)).argsort(1) < count[:, None]
        out = np.where(keep, np.clip(mag((n, 64)), -32767, 32767), 0)
    out = out.reshape(n, 8, 8)
    fix_dc_chain(out)
    return out


def fix_dc_chain(blocks: np.ndarray) -> None:
    """Nudges DC values (in place, [n, 8, 8] in coding order) so no DC difference is -32768 modulo 2^16, which no code has."""
    prev = 0
    for b in blocks:
        if ((int(b[0, 0]) - prev) & 0xFFFF) == 0x8000:
            b[0, 0] += 1 if b[0, 0] < 32767 else -1
        prev = int(b[0, 0])


def grey_file(blocks: np.ndarray, q: np.ndarray, cols: int, **kw) -> Written:
    """A grey file holding `blocks` ([n, 8, 8], coding order) `cols` blocks per row, zero blocks after them; `q` is table 0."""
    n = len(blocks)
    rows = -(-n // cols)
    grid = np.zeros((rows * cols, 8, 8), np.int64)
    grid[:n] = blocks
    return write_jpeg([grid.reshape(rows, cols, 8, 8)], {0: q}, height=rows * 8, width=cols * 8, sampling=[(1, 1)], **kw)


# ---------------------------------------------------------------------------------------------------------------------
# Decoder back end
# ---------------------------------------------------------------------------------------------------------------------
F_0_298, F_0_390, F_0_541, F_0_765, F_0_899, F_1_175 = 2446, 3196, 4433, 6270, 7373, 9633
F_1_501, F_1_847, F_1_961, F_2_053, F_2_562, F_3_072 = 12299, 15137, 16069, 16819, 20995, 25172


def _w16(x):
    return ((x + 32768) & 0xFFFF) - 32768


def _idct_1d(d):
    """One 1-D pass of the SIMD islow over the last axis of int64 `d` (int16 values); 32-bit results (no overflow: every
    sum is bounded by 2^31 for 16-bit inputs)."""
    i0, i1, i2, i3, i4, i5, i6, i7 = (d[..., k] for k in range(8))
    tmp3 = i2 * (F_0_541 + F_0_765) + i6 * F_0_541
    tmp2 = i2 * F_0_541 + i6 * (F_0_541 - F_1_847)
    tmp0 = _w16(i0 + i4) * 8192
    tmp1 = _w16(i0 - i4) * 8192
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    z3 = _w16(i7 + i3)
    z4 = _w16(i5 + i1)
    z3p = z3 * (F_1_175 - F_1_961) + z4 * F_1_175
    z4p = z3 * F_1_175 + z4 * (F_1_175 - F_0_390)
    o0 = i7 * (F_0_298 - F_0_899) + i1 * -F_0_899 + z3p
    o3 = i7 * -F_0_899 + i1 * (F_1_501 - F_0_899) + z4p
    o1 = i5 * (F_2_053 - F_2_562) + i3 * -F_2_562 + z4p
    o2 = i5 * -F_2_562 + i3 * (F_3_072 - F_2_562) + z3p
    return np.stack([tmp10 + o3, tmp11 + o2, tmp12 + o1, tmp13 + o0, tmp13 - o0, tmp12 - o1, tmp11 - o2, tmp10 - o3], -1)


def idct_islow_simd(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """uint8 [N, 8, 8] from int [N, 8, 8] coefficients (natural order, int16 range) and a natural-order table (uint16)."""
    coef = np.asarray(coef, np.int64).reshape(-1, 8, 8)
    w = _w16(coef * np.asarray(q, np.int64).reshape(8, 8))          # pmullw: low 16 bits of the product
    p1 = np.clip((_idct_1d(w.transpose(0, 2, 1)) + 1024) >> 11, -32768, 32767).transpose(0, 2, 1)   # columns, packssdw
    dc_only = ~np.any(coef[:, 1:, :] != 0, axis=(1, 2))             # rows 1-7 of the whole block zero
    p1[dc_only] = _w16(w[dc_only, 0:1, :] * 4)                      # psllw: row 0 shifted, 16-bit, for every row
    p2 = (_idct_1d(p1) + (1 << 17)) >> 18                           # rows
    return (np.clip(p2, -128, 127) + 128).astype(np.uint8)          # packssdw, packsswb, + CENTERJSAMPLE


def _upsample(pl: np.ndarray, h: int, w: int, hs: int, vs: int, dw: int, dh: int) -> np.ndarray:
    """jdsample.c / jdsample-*.asm as jinit_upsampler picks them with fancy upsampling on."""
    pl = pl.astype(np.int64)
    ys, xs = np.arange(h)[:, None], np.arange(w)[None, :]
    if (hs, vs) == (1, 1):
        return pl[:h, :w]
    if (hs, vs) == (2, 1):
        j = xs >> 1
        if dw <= 2:
            return pl[ys, j]
        jn = np.where(xs & 1, np.minimum(j + 1, dw - 1), np.maximum(j - 1, 0))
        return (3 * pl[ys, j] + pl[ys, jn] + 1 + (xs & 1)) >> 2
    if (hs, vs) == (1, 2):
        i = ys >> 1
        inn = np.where(ys & 1, np.minimum(i + 1, dh - 1), np.maximum(i - 1, 0))
        return (3 * pl[i, xs] + pl[inn, xs] + 1 + (ys & 1)) >> 2
    if (hs, vs) == (2, 2):
        i, j = ys >> 1, xs >> 1
        if dw <= 2:
            return pl[i, j]
        inn = np.where(ys & 1, np.minimum(i + 1, dh - 1), np.maximum(i - 1, 0))
        jn = np.where(xs & 1, np.minimum(j + 1, dw - 1), np.maximum(j - 1, 0))
        c0 = 3 * pl[i, j] + pl[inn, j]
        c1 = 3 * pl[i, jn] + pl[inn, jn]
        return (3 * c0 + c1 + 8 - (xs & 1)) >> 4
    assert (hs, vs) == (4, 1)
    return pl[ys, xs >> 2]


def decode_coefs(coefs: Sequence[np.ndarray], qt: Sequence[np.ndarray], height: int, width: int,
                 sampling: Sequence[Tuple[int, int]]) -> np.ndarray:
    """HWC uint8 RGB, as Helper._read_img returns it (grey as three equal channels), from the coefficients a Huffman decode
    yields (absolute DC, int16) and the quantisation tables latched at the scan."""
    planes = []
    for c, q in zip(coefs, qt):
        c = np.asarray(c, np.int64)
        gh, gw = c.shape[:2]
        planes.append(idct_islow_simd(c.reshape(-1, 8, 8), q).reshape(gh, gw, 8, 8).transpose(0, 2, 1, 3).reshape(gh * 8, gw * 8))
    y = planes[0][:height, :width].astype(np.int64)
    if len(planes) == 1:
        return np.repeat(y[..., None].astype(np.uint8), 3, -1)
    hmax = max(h for h, _ in sampling)
    vmax = max(v for _, v in sampling)
    hs, vs = hmax // sampling[1][0], vmax // sampling[1][1]
    dw, dh = -(-width * sampling[1][0] // hmax), -(-height * sampling[1][1] // vmax)
    cb = _upsample(planes[1], height, width, hs, vs, dw, dh) - 128
    cr = _upsample(planes[2], height, width, hs, vs, dw, dh) - 128
    r = y + ((91881 * cr + 32768) >> 16)
    g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)
