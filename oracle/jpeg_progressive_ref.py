"""TEST INFRASTRUCTURE — a plain-Python progressive Huffman JPEG entropy decoder (SOF2): file bytes in, quantised
coefficients out, for ``jpeg_ref.decode_coefs`` to turn into pixels.

Only tests/ may import this module; the product path is k210_yolo_framework_b200/csrc/jpeg_progressive.cu.

Written from ITU T.81 (G.1.2 progressive Huffman decoding) and the behaviour of the libjpeg-turbo decoder PIL runs:
- the four scan kinds: DC first (differences of the values shifted right by Al, each sum stored as the int16 of
  ``(unsigned)v << Al``), DC refinement (one raw bit per block), AC first (runs, ZRL, EOBn runs) and AC refinement
  (correction bits of the nonzero coefficients, new +-1 << Al coefficients whatever the symbol's size, EOBn runs);
- a run may end past the scan's band: the decoder indexes the natural order at k, and the natural order continues past
  zig-zag 63 with sixteen more entries of 63, so an AC first scan writes zig-zag min(k, 63) for k up to Se + 15 and an AC
  refinement writes zig-zag Se + 1 (or 63) when its zero run leaves the band;
- each restart interval starts with the DC predictions and the EOB run at zero and the bit reader at the next segment;
- bytes: 0xFF 0x00 is a data 0xFF, 0xFF bytes before another 0xFF are fill, 0xFF then 0xD0..0xD7 is a restart marker, any
  other marker ends the scan's data.  Bits read past a segment's end are zeros, and the rest of that interval is left as it
  is (libjpeg's insufficient-data rule); `Decoded.hit_end` lists the intervals where that happened;
- scans are decoded in file order.  Restart markers out of sequence are reported (`Decoded.restart_issues`), not modelled:
  libjpeg-turbo's resynchronisation then drops or rereads data, and the coefficients here are the in-order reading only.

Quantisation tables are latched at each component's first scan.  Arithmetic coding and block smoothing are not modelled.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle.jpeg_ref import ZIGZAG

NATURAL_EXT = [int(z) for z in ZIGZAG] + [63] * 16     # zig-zag index -> natural position, 16 entries past the end


@dataclasses.dataclass
class Scan:
    comps: List[int]
    ss: int
    se: int
    ah: int
    al: int
    restart: int
    markers: List[int]           # numbers n of the RSTn markers in the scan's data, in file order


@dataclasses.dataclass
class Decoded:
    coefs: List[np.ndarray]      # per frame component int16 [bh, bw, 8, 8] natural order (jpeg_ref.block_grid size)
    qt: List[np.ndarray]         # per frame component, natural order, as latched at its first scan
    sampling: List[Tuple[int, int]]
    height: int
    width: int
    scans: List[Scan]
    restart_issues: List[str]    # markers out of sequence, missing, or present with no restart interval
    hit_end: List[Tuple[int, int]]   # (scan, interval) that read bits past its data


def _i16(v: int) -> int:
    return ((v + 32768) & 0xFFFF) - 32768


class _Bits:
    """MSB-first bits of one restart segment (stuffing and fill bytes dropped), zeros past its end."""

    def __init__(self, data: bytes):
        self.data, self.pos, self.bit, self.past = data, 0, 0, False

    def get(self, n: int) -> int:
        v = 0
        for _ in range(n):
            if self.pos < len(self.data):
                b = (self.data[self.pos] >> (7 - self.bit)) & 1
                self.bit += 1
                if self.bit == 8:
                    self.pos, self.bit = self.pos + 1, 0
            else:
                b, self.past = 0, True
            v = (v << 1) | b
        return v

    def huff(self, table: Dict[Tuple[int, int], int]) -> int:
        code = 0
        for length in range(1, 17):
            code = (code << 1) | self.get(1)
            if (length, code) in table:
                return table[(length, code)]
        raise ValueError("invalid Huffman code")


def _extend(v: int, s: int) -> int:
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def _huff_table(bits: List[int], vals: List[int]) -> Dict[Tuple[int, int], int]:
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[(length, code)] = vals[k]
            code, k = code + 1, k + 1
        code <<= 1
    return out


def _segments(d: bytes, at: int) -> Tuple[List[bytes], List[int], int]:
    """The scan's entropy-coded data from `at`: unstuffed bytes of each restart segment, the marker numbers between them,
    and the offset of the marker that ends the data."""
    segs, markers, cur, i = [], [], bytearray(), at
    while i < len(d):
        b = d[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        j = i + 1
        while j < len(d) and d[j] == 0xFF:
            j += 1
        nx = d[j] if j < len(d) else 0xD9
        if nx == 0x00:
            cur.append(0xFF)
            i = j + 1
        elif 0xD0 <= nx <= 0xD7:
            segs.append(bytes(cur))
            markers.append(nx - 0xD0)
            cur = bytearray()
            i = j + 1
        else:
            i = j - 1 if j > i + 1 else i   # the marker's own 0xFF
            break
    segs.append(bytes(cur))
    return segs, markers, i


def _scan_blocks(comps, hs, vs, height, width) -> List[List[Tuple[int, int, int]]]:
    """(component, block row, block column) of each MCU of a scan."""
    n = len(hs)
    hmax, vmax = (max(hs), max(vs)) if n > 1 else (1, 1)
    if len(comps) == 1:
        c = comps[0]
        hc, vc = (hs[c], vs[c]) if n > 1 else (1, 1)
        dw, dh = -(-width * hc // hmax), -(-height * vc // vmax)
        return [[(c, r, q)] for r in range(-(-dh // 8)) for q in range(-(-dw // 8))]
    mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    return [[(c, y * vs[c] + j, x * hs[c] + i) for c in comps for j in range(vs[c]) for i in range(hs[c])]
            for y in range(my) for x in range(mx)]


def decode(data: bytes) -> Decoded:
    d = bytes(data)
    if d[:2] != b"\xff\xd8":
        raise ValueError("not a JPEG file")
    i = 2
    qt: Dict[int, np.ndarray] = {}
    dc_tabs: Dict[int, Dict] = {}
    ac_tabs: Dict[int, Dict] = {}
    restart = 0
    frame = None
    coefs: List[np.ndarray] = []
    latched: Dict[int, np.ndarray] = {}
    scans: List[Scan] = []
    issues: List[str] = []
    hit_end: List[Tuple[int, int]] = []
    while True:
        while i < len(d) and d[i] == 0xFF and i + 1 < len(d) and d[i + 1] == 0xFF:
            i += 1
        if i + 1 >= len(d) or d[i] != 0xFF:
            raise ValueError(f"no marker at offset {i}")
        m = d[i + 1]
        if m == 0xD9:
            break
        if 0xD0 <= m <= 0xD7:       # a stray marker between scans: parameterless
            i += 2
            continue
        ln = int.from_bytes(d[i + 2:i + 4], "big")
        p = d[i + 4:i + 2 + ln]
        nxt = i + 2 + ln
        if m == 0xDB:
            k = 0
            while k < len(p):
                prec, tid = p[k] >> 4, p[k] & 15
                w = 2 if prec else 1
                vals = [int.from_bytes(p[k + 1 + w * z:k + 1 + w * z + w], "big") for z in range(64)]
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = vals
                qt[tid] = q
                k += 1 + 64 * w
        elif m == 0xC4:
            k = 0
            while k < len(p):
                cls, tid = p[k] >> 4, p[k] & 15
                bits = list(p[k + 1:k + 17])
                vals = list(p[k + 17:k + 17 + sum(bits)])
                (ac_tabs if cls else dc_tabs)[tid] = _huff_table(bits, vals)
                k += 17 + sum(bits)
        elif m == 0xDD:
            restart = int.from_bytes(p[:2], "big")
        elif m == 0xC2:
            height, width, n = int.from_bytes(p[1:3], "big"), int.from_bytes(p[3:5], "big"), p[5]
            ids = [p[6 + 3 * c] for c in range(n)]
            hs = [p[7 + 3 * c] >> 4 for c in range(n)]
            vs = [p[7 + 3 * c] & 15 for c in range(n)]
            tq = [p[8 + 3 * c] for c in range(n)]
            frame = (height, width, ids, hs, vs, tq)
            hmax, vmax = (max(hs), max(vs)) if n > 1 else (1, 1)
            mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
            grid = [(my * (vs[c] if n > 1 else 1), mx * (hs[c] if n > 1 else 1)) for c in range(n)]
            coefs = [np.zeros((gh, gw, 64), np.int64) for gh, gw in grid]
        elif m == 0xDA:
            assert frame is not None, "SOS before SOF2"
            height, width, ids, hs, vs, tq = frame
            ns = p[0]
            comps = [ids.index(p[1 + 2 * k]) for k in range(ns)]
            tsel = [(p[2 + 2 * k] >> 4, p[2 + 2 * k] & 15) for k in range(ns)]
            ss, se, ah, al = p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns] >> 4, p[3 + 2 * ns] & 15
            for c in comps:
                latched.setdefault(c, qt[tq[c]].copy())
            segs, markers, end = _segments(d, nxt)
            si = len(scans)
            scans.append(Scan(comps, ss, se, ah, al, restart, markers))
            mcus = _scan_blocks(comps, hs, vs, height, width)
            per = restart if restart else len(mcus)
            nint = -(-len(mcus) // per) if mcus else 0
            if not restart and markers:
                issues.append(f"scan {si}: RST{markers[0]} with no restart interval")
            if restart:
                for k, num in enumerate(markers[:max(nint - 1, 0)]):
                    if num != k % 8:
                        issues.append(f"scan {si}: restart marker {k} is RST{num}, not RST{k % 8}")
                        break
                if len(markers) < nint - 1:
                    issues.append(f"scan {si}: {len(markers)} restart markers of {nint - 1}")
            tabs = {c: (dc_tabs.get(td), ac_tabs.get(ta)) for c, (td, ta) in zip(comps, tsel)}
            for k in range(nint):
                br = _Bits(segs[k] if k < len(segs) else b"")
                _decode_interval(br, mcus[k * per:(k + 1) * per], coefs, tabs, ss, se, ah, al)
                if br.past:
                    hit_end.append((si, k))
            nxt = end
        elif m in (0xC0, 0xC1, 0xC3) or 0xC5 <= m <= 0xCF and m != 0xC8 and m != 0xCC:
            raise ValueError(f"not a progressive Huffman file (SOF 0x{m:02X})")
        i = nxt
    height, width, ids, hs, vs, tq = frame
    n = len(ids)
    out = []
    for c in range(n):
        gh, gw = coefs[c].shape[:2]
        out.append(coefs[c].reshape(gh, gw, 8, 8).astype(np.int16))
    samp = [(hs[c], vs[c]) for c in range(n)] if n > 1 else [(1, 1)]
    return Decoded(out, [latched.get(c, np.zeros(64, np.int64)) for c in range(n)], samp, height, width, scans, issues,
                   hit_end)


def _decode_interval(br: _Bits, mcus, coefs, tabs, ss, se, ah, al) -> None:
    pred: Dict[int, int] = {}
    eobrun = 0
    p1, m1 = 1 << al, -(1 << al)
    for mcu in mcus:
        if br.past:              # libjpeg leaves the rest of an interval that ran out of data as it is
            return
        for c, by, bx in mcu:
            blk = coefs[c][by, bx]
            if ss == 0 and ah == 0:
                s = br.huff(tabs[c][0])
                v = pred.get(c, 0) + (_extend(br.get(s), s) if s else 0)
                if not -2 ** 31 <= v < 2 ** 31:
                    raise ValueError("DC value outside int")
                pred[c] = v
                blk[0] = _i16((v & 0xFFFFFFFF) << al)
            elif ss == 0:
                if br.get(1):
                    blk[0] = _i16(int(blk[0]) | p1)
            elif ah == 0:
                if eobrun:
                    eobrun -= 1
                    continue
                k = ss
                while k <= se:
                    rs = br.huff(tabs[c][1])
                    r, s = rs >> 4, rs & 15
                    if s:
                        k += r
                        blk[NATURAL_EXT[k]] = _i16((_extend(br.get(s), s) & 0xFFFFFFFF) << al)
                    elif r == 15:
                        k += 15
                    else:
                        eobrun = (1 << r) + (br.get(r) if r else 0) - 1
                        break
                    k += 1
            else:
                k = ss
                if eobrun == 0:
                    while k <= se:
                        rs = br.huff(tabs[c][1])
                        r, s = rs >> 4, rs & 15
                        if s:
                            s = p1 if br.get(1) else m1
                        elif r != 15:
                            eobrun = 1 << r
                            if r:
                                eobrun += br.get(r)
                            break
                        while k <= se:
                            pos = NATURAL_EXT[k]
                            if blk[pos] != 0:
                                if br.get(1) and (int(blk[pos]) & p1) == 0:
                                    blk[pos] = _i16(int(blk[pos]) + (p1 if blk[pos] >= 0 else m1))
                            else:
                                r -= 1
                                if r < 0:
                                    break
                            k += 1
                        if s:
                            blk[NATURAL_EXT[k]] = s
                        k += 1
                if eobrun > 0:
                    while k <= se:
                        pos = NATURAL_EXT[k]
                        if blk[pos] != 0 and br.get(1) and (int(blk[pos]) & p1) == 0:
                            blk[pos] = _i16(int(blk[pos]) + (p1 if blk[pos] >= 0 else m1))
                        k += 1
                    eobrun -= 1


def decode_pixels(data: bytes) -> np.ndarray:
    """HWC uint8 RGB through ``jpeg_ref.decode_coefs``."""
    from oracle.jpeg_ref import decode_coefs
    r = decode(data)
    return decode_coefs(r.coefs, r.qt, r.height, r.width, r.sampling)
