"""TEST INFRASTRUCTURE — a progressive Huffman JPEG writer (SOF2) with an arbitrary scan script, after libjpeg-turbo's
jcphuff.c, built on oracle/jpeg_ref.py's tables and bit packing.  PIL writes progressive files only with libjpeg's default
script; this writer is how the tests get spectral selection, successive approximation and restart intervals in any
combination, including scripts libjpeg-turbo only warns about.

`write_progressive(coefs, qtables, height=, width=, sampling=, script=)`: `coefs` per frame component [bh, bw, 8, 8] in
natural order (MCU-padded, ``jpeg_ref.block_grid``), absolute DC.  `script`: scans (components, Ss, Se, Ah, Al).  Each scan
is encoded as jcphuff.c encodes it: DC first as differences of the values shifted right by Al, DC refine as one raw bit,
AC first with EOBn runs, AC refine with its correction bits buffered until the next symbol or EOB run (forced out past
jcphuff.c's MAX_CORR_BITS).  EOB runs end at each restart marker and at the end of the scan.  `restart`: one interval for
every scan or one per scan (a DRI marker goes before each scan whose interval differs from the one in force).  `huffman`:
"optimal" (jpeg_gen_optimal_table per scan, as libjpeg-turbo's progressive mode does) or "flat" (every symbol a scan uses
at one length).  Each scan's tables are defined by a DHT right before its SOS.

`write_scans(qtables, height=, width=, sampling=, scans=)` writes a frame from explicit entropy-coded items instead: per scan
and restart segment, the Huffman symbols and raw bit fields `_Seg` holds, with tables built from the symbols each scan uses
(or given), any RSTn numbering, markers left out or added, fill bytes before markers and in the data, and zero padding.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple, Union

import numpy as np

from oracle import jpeg_ref as J

MAX_CORR_BITS = 1000   # jcphuff.c

# jcparam.c jpeg_simple_progression
DEFAULT_SCRIPT_YCC = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((0,), 6, 63, 0, 2),
                      ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
DEFAULT_SCRIPT_GREY = [((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
                       ((0,), 1, 63, 1, 0)]


def _ashr(v: int, s: int) -> int:
    return int(v) >> s      # IRIGHT_SHIFT: arithmetic


def _scan_mcus(coefs, comps, sampling, height, width):
    """The blocks of each MCU of a scan, as [(table index, component, by, bx)] lists."""
    if len(comps) == 1:
        c = comps[0]
        if len(sampling) == 1:
            rows, cols = -(-height // 8), -(-width // 8)
        else:
            hmax = max(h for h, _ in sampling)
            vmax = max(v for _, v in sampling)
            dw, dh = -(-width * sampling[c][0] // hmax), -(-height * sampling[c][1] // vmax)
            rows, cols = -(-dh // 8), -(-dw // 8)
        return [[(0, c, r, q)] for r in range(rows) for q in range(cols)]
    hmax = max(h for h, _ in sampling)
    vmax = max(v for _, v in sampling)
    mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    out = []
    for y in range(my):
        for x in range(mx):
            mcu = []
            for k, c in enumerate(comps):
                hs, vs = sampling[c]
                mcu += [(k, c, y * vs + by, x * hs + bx) for by in range(vs) for bx in range(hs)]
            out.append(mcu)
    return out


class _Seg:
    """Items of one restart segment: ("s", table, symbol) or ("b", value, nbits)."""

    def __init__(self):
        self.items: List[Tuple] = []
        self.eobrun = 0
        self.be: List[int] = []     # correction bits buffered behind the pending EOB run

    def sym(self, t, s):
        self.items.append(("s", t, s))

    def bits(self, v, n):
        if n:
            self.items.append(("b", int(v) & ((1 << n) - 1), n))

    def emit_eobrun(self):
        if self.eobrun > 0:
            nbits = self.eobrun.bit_length() - 1
            assert nbits <= 14
            self.sym(0, nbits << 4)
            self.bits(self.eobrun, nbits)
            self.eobrun = 0
            for b in self.be:
                self.bits(b, 1)
            self.be = []


def _encode_segment(blocks, mcus, ss, se, ah, al) -> _Seg:
    seg = _Seg()
    last_dc: Dict[int, int] = {}
    for mcu in mcus:
        for t, c, by, bx in mcu:
            blk = blocks[c][by, bx].reshape(64)
            if ss == 0 and ah == 0:
                v = _ashr(blk[0], al)
                diff = v - last_dc.get(c, 0)
                last_dc[c] = v
                n = J._category(diff)
                seg.sym(t, n)
                seg.bits(J._magnitude_bits(diff, n), n)
            elif ss == 0:
                seg.bits(_ashr(blk[0], al) & 1, 1)
            elif ah == 0:
                r = 0
                for k in range(ss, se + 1):
                    v = int(blk[J.ZIGZAG[k]])
                    a = (-v if v < 0 else v) >> al
                    if a == 0:
                        r += 1
                        continue
                    seg.emit_eobrun()
                    while r > 15:
                        seg.sym(0, 0xF0)
                        r -= 16
                    n = a.bit_length()
                    seg.sym(0, (r << 4) + n)
                    seg.bits(a if v >= 0 else ~a, n)
                    r = 0
                if r > 0:
                    seg.eobrun += 1
                    if seg.eobrun == 0x7FFF:
                        seg.emit_eobrun()
            else:
                absv = {k: (abs(int(blk[J.ZIGZAG[k]])) >> al) for k in range(ss, se + 1)}
                eob = max([k for k in absv if absv[k] == 1], default=0)
                r, br = 0, []
                for k in range(ss, se + 1):
                    a = absv[k]
                    if a == 0:
                        r += 1
                        continue
                    while r > 15 and k <= eob:
                        seg.emit_eobrun()
                        seg.sym(0, 0xF0)
                        r -= 16
                        for b in br:
                            seg.bits(b, 1)
                        br = []
                    if a > 1:
                        br.append(a & 1)
                        continue
                    seg.emit_eobrun()
                    seg.sym(0, (r << 4) + 1)
                    seg.bits(0 if blk[J.ZIGZAG[k]] < 0 else 1, 1)
                    for b in br:
                        seg.bits(b, 1)
                    br = []
                    r = 0
                if r > 0 or br:
                    seg.eobrun += 1
                    seg.be += br
                    if seg.eobrun == 0x7FFF or len(seg.be) > MAX_CORR_BITS - 64 + 1:
                        seg.emit_eobrun()
    seg.emit_eobrun()
    return seg


def write_progressive(coefs: Sequence[np.ndarray], qtables: Dict[int, np.ndarray], *, height: int, width: int,
                      sampling: Sequence[Tuple[int, int]], script: Sequence[Tuple[Sequence[int], int, int, int, int]],
                      tq: Sequence[int] = None, restart: Union[int, Sequence[int]] = 0, huffman: str = "optimal",
                      ids: Sequence[int] = None, jfif: bool = True) -> bytes:
    n = len(coefs)
    tq = list(tq) if tq is not None else [0] + [1] * (n - 1)
    ids = list(ids) if ids is not None else list(range(1, n + 1))
    restarts = [restart] * len(script) if isinstance(restart, int) else list(restart)
    blocks = [np.asarray(c, np.int64) for c in coefs]
    out = b"\xff\xd8"
    if jfif:
        out += J._segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    qt = {t: np.asarray(q, np.int64).reshape(64) for t, q in qtables.items()}
    out += J._segment(0xDB, J._dqt(qt, {t: int(q.max() > 255) for t, q in qt.items()}))
    sof = bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([n])
    for c in range(n):
        sof += bytes([ids[c], (sampling[c][0] << 4) | sampling[c][1], tq[c]])
    out += J._segment(0xC2, sof)
    dri = 0
    for (comps, ss, se, ah, al), rst in zip(script, restarts):
        comps = list(comps)
        mcus = _scan_mcus(blocks, comps, sampling, height, width)
        per = rst if rst else len(mcus)
        segs = [_encode_segment(blocks, mcus[i:i + per], ss, se, ah, al) for i in range(0, len(mcus), per)]
        ntab = len(comps) if ss == 0 else 1
        cls = "dc" if ss == 0 else "ac"
        freq = [dict() for _ in range(ntab)]
        for s in segs:
            for it in s.items:
                if it[0] == "s":
                    freq[it[1]][it[2]] = freq[it[1]].get(it[2], 0) + 1
        htabs = {}
        if not (ss == 0 and ah != 0):
            for t in range(ntab):
                f = freq[t] or {0: 1}
                if huffman == "optimal":
                    htabs[(cls, t)] = J.optimal_table(f)
                else:
                    htabs[(cls, t)] = J.flat_table(sorted(f), max(1, len(f).bit_length()))
            out += J._segment(0xC4, J._dht(htabs))
        if rst != dri:
            out += J._segment(0xDD, rst.to_bytes(2, "big"))
            dri = rst
        sos = bytes([len(comps)])
        for k, c in enumerate(comps):
            sos += bytes([ids[c], (k << 4) if ss == 0 else 0])
        sos += bytes([ss, se, (ah << 4) | al])
        out += J._segment(0xDA, sos)
        codes = {t: J._codes(htabs[(cls, t)]) for t in range(ntab)} if htabs else {}
        for si, s in enumerate(segs):
            words = [(codes[t][sym][0], codes[t][sym][1]) if kind == "s" else (t, sym) for kind, t, sym in s.items]
            w = np.array([a for a, _ in words], np.int64)
            ln = np.array([b for _, b in words], np.int64)
            bits = J._bit_array(w, ln)
            bits = np.concatenate([bits, np.ones((-len(bits)) % 8, np.uint8)])
            out += J._stuff(bits)
            if si + 1 < len(segs):
                out += bytes([0xFF, 0xD0 + si % 8])
    return out + b"\xff\xd9"


def known_coefs(coefs: Sequence[np.ndarray], script, ncomp: int) -> List[np.ndarray]:
    """What a decoder holds after `script`: each coefficient down to the last Al its scans sent (zero if never sent), the
    rounding toward zero successive approximation gives (DC: floor, as jcphuff.c shifts it arithmetically)."""
    al = np.full((ncomp, 64), -1)
    for comps, ss, se, ah, a in script:
        for c in comps:
            for k in range(ss, se + 1):
                al[c, J.ZIGZAG[k]] = a
    out = []
    for c in range(ncomp):
        x = np.asarray(coefs[c], np.int64).reshape(-1, 64).copy()
        for pos in range(64):
            if al[c, pos] < 0:
                x[:, pos] = 0
            elif pos == 0:
                x[:, 0] = (x[:, 0] >> al[c, 0]) << al[c, 0]
            else:
                s = al[c, pos]
                x[:, pos] = np.sign(x[:, pos]) * ((np.abs(x[:, pos]) >> s) << s)
        out.append(x.reshape(np.asarray(coefs[c]).shape))
    return out


def write_scans(qtables: Dict[int, np.ndarray], *, height: int, width: int, sampling: Sequence[Tuple[int, int]],
                scans: Sequence[dict], tq: Sequence[int] = None, ids: Sequence[int] = None, jfif: bool = True) -> bytes:
    """A progressive file from explicit entropy-coded items, for bitstreams jcphuff.c never writes.

    Each scan is a dict: ``comps``, ``ss``, ``se``, ``ah``, ``al`` as in a script entry; ``segs``: one item list per restart
    segment, items ("s", table, symbol) (table: index of the component in a DC first scan, else 0) or ("b", value, nbits)
    as ``_Seg`` holds them; optional:
      huffman  "flat" (default), "optimal", or {table: (bits, values)}; a DHT with the scan's tables goes right before its SOS
      restart  the DRI interval in force (a DRI marker goes before the scan when it differs from the one in force; default 0)
      markers  the number n of the RSTn written after each segment but the last (default k % 8), None to leave a marker out
      extra    the number of one more RSTn after the last segment (default none)
      pad      "ones" (default) or "zeros" to the byte boundary at each segment's end
      fill     0xFF fill bytes before each RSTn and before the next marker after the scan
      fill_data  0xFF fill bytes before each stuffed 0xFF 0x00 in the data
    """
    n = len(sampling)
    tq = list(tq) if tq is not None else [0] + [1] * (n - 1)
    ids = list(ids) if ids is not None else list(range(1, n + 1))
    out = b"\xff\xd8"
    if jfif:
        out += J._segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    qt = {t: np.asarray(q, np.int64).reshape(64) for t, q in qtables.items()}
    out += J._segment(0xDB, J._dqt(qt, {t: int(q.max() > 255) for t, q in qt.items()}))
    sof = bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([n])
    for c in range(n):
        sof += bytes([ids[c], (sampling[c][0] << 4) | sampling[c][1], tq[c]])
    out += J._segment(0xC2, sof)
    dri = 0
    for sc in scans:
        comps, ss, se, ah, al = list(sc["comps"]), sc["ss"], sc["se"], sc["ah"], sc["al"]
        segs = sc["segs"]
        ntab = len(comps) if ss == 0 else 1
        cls = "dc" if ss == 0 else "ac"
        htabs = {}
        if not (ss == 0 and ah != 0):
            freq = [dict() for _ in range(ntab)]
            for items in segs:
                for it in items:
                    if it[0] == "s":
                        freq[it[1]][it[2]] = freq[it[1]].get(it[2], 0) + 1
            huff = sc.get("huffman", "flat")
            for t in range(ntab):
                f = freq[t] or {0: 1}
                if isinstance(huff, dict):
                    htabs[(cls, t)] = huff[t]
                elif huff == "optimal":
                    htabs[(cls, t)] = J.optimal_table(f)
                else:
                    htabs[(cls, t)] = J.flat_table(sorted(f), max(1, len(f).bit_length()))
            out += J._segment(0xC4, J._dht(htabs))
        rst = sc.get("restart", 0)
        if rst != dri:
            out += J._segment(0xDD, rst.to_bytes(2, "big"))
            dri = rst
        sos = bytes([len(comps)])
        for k, c in enumerate(comps):
            sos += bytes([ids[c], (k << 4) if ss == 0 else 0])
        out += J._segment(0xDA, sos + bytes([ss, se, (ah << 4) | al]))
        codes = {t: J._codes(htabs[(cls, t)]) for t in range(ntab)} if htabs else {}
        markers = sc.get("markers") or [k % 8 for k in range(len(segs) - 1)]
        fill, pad = b"\xff" * sc.get("fill", 0), sc.get("pad", "ones")
        for si, items in enumerate(segs):
            words = [codes[t][sym] if kind == "s" else (t, sym) for kind, t, sym in items]
            bits = J._bit_array(np.array([a for a, _ in words], np.int64), np.array([b for _, b in words], np.int64))
            npad = (-len(bits)) % 8
            bits = np.concatenate([bits, np.ones(npad, np.uint8) if pad == "ones" else np.zeros(npad, np.uint8)])
            data = J._stuff(bits)
            if sc.get("fill_data"):
                data = data.replace(b"\xff\x00", b"\xff" * sc["fill_data"] + b"\xff\x00")
            out += data
            num = markers[si] if si + 1 < len(segs) else sc.get("extra")
            if num is not None:
                out += fill + bytes([0xFF, 0xD0 + num])
        out += fill
    return out + b"\xff\xd9"
