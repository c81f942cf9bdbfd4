"""TEST INFRASTRUCTURE — progressive (and a few baseline) JPEG files with bitstreams libjpeg-turbo's compressor never writes,
built item by item with ``progressive_writer.write_scans`` or by renumbering, dropping and adding restart markers in PIL's
own files.

``exact_cases()``: files libjpeg-turbo decodes without resynchronising, whose coefficients ``oracle.jpeg_progressive_ref``
gives: runs that end past their scan's band (AC first scans to Se + 1 .. Se + 15 and past zig-zag 63, AC refinements to
Se + 1) in both orders against the scan that owns the coefficient, with restart intervals and 4:2:0 colour; ZRL before EOB and
past Se; refinement symbols of sizes 2, 7 and 15; EOB runs of 32767 and runs longer than the blocks left; 16-bit codes, one-symbol
tables, a table redefined between two scans of one level; DC at Al 13; DC refinements over intervals that are not multiples
of 16 blocks; fill bytes and zero padding.

``resync_cases()`` / ``baseline_resync_cases()``: files whose restart markers are out of sequence (renumbered by +1, +2,
-1, -2, +4, one left out, one added, one inside a scan with no restart interval).  libjpeg-turbo resynchronises on them;
a GPU decoder must give PIL's pixels or refuse the file.
"""
from __future__ import annotations

import io
from typing import List, Tuple

import numpy as np

import progressive_writer as W
from oracle import jpeg_ref as J

Q4 = np.full(64, 4, np.int64)


def S(sym, t=0):
    return ("s", t, sym)


def B(v, n):
    return ("b", v & ((1 << n) - 1), n)


def dc(v):
    """A DC first symbol and value for a difference v."""
    s = J._category(v)
    return [S(s)] + ([B(J._magnitude_bits(v, s), s)] if s else [])


EOB = S(0x00)
ZRL = S(0xF0)


def scan(comps, ss, se, ah, al, *segs, **kw):
    return dict(comps=comps, ss=ss, se=se, ah=ah, al=al, segs=list(segs), **kw)


def grey(scans, blocks=(1, 1)):
    """A grey file of `blocks` (rows, cols) 8x8 blocks, quantiser 4 everywhere."""
    return W.write_scans({0: Q4}, height=8 * blocks[0], width=8 * blocks[1], sampling=[(1, 1)], scans=scans)


DC5 = scan((0,), 0, 0, 0, 0, dc(5))


def _stray_cases() -> List[Tuple[str, bytes]]:
    out = []
    # AC refinement past Se, then the first scan that owns the coefficient: zz6 = 7 in file order
    out.append(("refine-stray-then-owner", grey([
        DC5, scan((0,), 1, 5, 0, 1, [S(0x01), B(1, 1), EOB]),
        scan((0,), 1, 5, 1, 0, [S(0x41), B(1, 1), B(0, 1)]),
        scan((0,), 6, 63, 0, 0, [S(0x03), B(7, 3), EOB])])))
    # AC first past Se after the owner: zz7 = 3 overwrites 9
    out.append(("first-stray-after-owner", grey([
        DC5, scan((0,), 6, 63, 0, 0, [S(0x14), B(9, 4), EOB]), scan((0,), 1, 5, 0, 0, [S(0x62), B(3, 2)])])))
    # AC first to Se + 15 (band 5..5, ZRL-sized run with a value), before and after the owner of zz20
    out.append(("first-stray-se15-before-owner", grey([
        DC5, scan((0,), 1, 4, 0, 0, [EOB]), scan((0,), 5, 5, 0, 0, [S(0xF2), B(2, 2)]),
        scan((0,), 6, 63, 0, 0, [S(0xE3), B(6, 3), EOB])])))
    out.append(("first-stray-se15-after-owner", grey([
        DC5, scan((0,), 1, 4, 0, 0, [EOB]), scan((0,), 6, 63, 0, 0, [S(0xE3), B(6, 3), EOB]),
        scan((0,), 5, 5, 0, 0, [S(0xF2), B(2, 2)])])))
    # every reach Se + 1 .. Se + 15 of a band 1..2 run, into the band of a 3..63 first scan written before it (zz7 = -2)
    for d in range(1, 16):
        out.append((f"first-stray-se{d}", grey([
            DC5, scan((0,), 3, 63, 0, 0, [S(0x42), B(1, 2), EOB]),
            scan((0,), 1, 2, 0, 0, [S(0x01), B(1, 1), S((d << 4) | 2), B(3, 2)])])))
    # past zig-zag 63: band 1..49 reaches k = 64 -> coefficient 63, before and after the owner writes it
    zrl3 = [ZRL, ZRL, ZRL]
    out.append(("first-stray-k64-before-owner", grey([
        DC5, scan((0,), 1, 49, 0, 0, zrl3 + [S(0xF2), B(2, 2)]), scan((0,), 50, 63, 0, 0, [S(0xD3), B(5, 3)])])))
    out.append(("first-stray-k64-after-owner", grey([
        DC5, scan((0,), 50, 63, 0, 0, [S(0xD3), B(5, 3)]), scan((0,), 1, 49, 0, 0, zrl3 + [S(0xF2), B(2, 2)])])))
    out.append(("first-k78-in-band", grey([
        DC5, scan((0,), 1, 62, 0, 0, [EOB]), scan((0,), 63, 63, 0, 0, [S(0xF3), B(4, 3)])])))
    # a stray into a band an earlier scan refined, and one into a band a later scan refines
    out.append(("stray-into-refined-band", grey([
        DC5, scan((0,), 6, 63, 0, 1, [S(0x01), B(1, 1), EOB]), scan((0,), 6, 63, 1, 0, [EOB, B(1, 1)]),
        scan((0,), 1, 5, 0, 0, [S(0x53), B(7, 3)])])))
    out.append(("stray-then-refined", grey([
        DC5, scan((0,), 1, 5, 0, 0, [S(0x52), B(2, 2)]), scan((0,), 6, 63, 0, 1, [EOB]),
        scan((0,), 6, 63, 1, 0, [EOB, B(1, 1)])])))
    # refinement to Se + 1 = 64 -> coefficient 63, in its own band
    out.append(("refine-stray-se63", grey([
        DC5, scan((0,), 1, 63, 0, 1, [S(0x01), B(1, 1), EOB]),
        scan((0,), 1, 63, 1, 0, [S(0xF1), B(1, 1), B(0, 1), S(0xF1), B(0, 1), S(0xE1), B(1, 1), S(0xF1), B(1, 1)])])))
    # the deterministic stray in every interval of a 2x3-block grey image, one block per interval
    segs1 = [[S(0x01), B(1, 1), EOB]] * 6
    segs2 = [[S(0x41), B(1, 1), B(0, 1)]] * 6
    segs3 = [[S(0x03), B(k + 1, 3), EOB] for k in range(6)]
    out.append(("refine-stray-restart1", grey([
        scan((0,), 0, 0, 0, 0, *[dc(k - 2) for k in range(6)], restart=1), scan((0,), 1, 5, 0, 1, *segs1, restart=1),
        scan((0,), 1, 5, 1, 0, *segs2, restart=1), scan((0,), 6, 63, 0, 0, *segs3, restart=1)], blocks=(2, 3))))
    # 4:2:0 colour, 16x16: four luma blocks, one of each chroma; the strays in luma and in Cr, restart every MCU in luma scans
    samp = [(2, 2), (1, 1), (1, 1)]
    ycc = [scan((0, 1, 2), 0, 0, 0, 0, dc(3) + dc(0) + dc(-1) + dc(2) + [S(1, 1), B(1, 1)] + [S(0, 2)])]
    ycc += [scan((0,), 1, 5, 0, 1, *[[S(0x01), B(1, 1), EOB]] * 4, restart=1),
            scan((0,), 1, 5, 1, 0, *[[S(0x41), B(1, 1), B(0, 1)]] * 4, restart=1),
            scan((0,), 6, 63, 0, 0, *[[S(0x03), B(5 - k, 3), EOB] for k in range(4)], restart=1),
            scan((1,), 1, 63, 0, 0, [EOB]), scan((2,), 6, 63, 0, 0, [S(0x14), B(9, 4), EOB]),
            scan((2,), 1, 5, 0, 0, [S(0x62), B(3, 2)])]
    out.append(("strays-420", W.write_scans({0: Q4, 1: Q4}, height=16, width=16, sampling=samp, scans=ycc)))
    return out


def _symbol_cases() -> List[Tuple[str, bytes]]:
    out = []
    full = [DC5]
    # ZRL then EOB, ZRL reaching past Se, in first and refinement scans
    out.append(("zrl-eob-first", grey(full + [scan((0,), 1, 63, 0, 0, [S(0x01), B(1, 1), ZRL, EOB])])))
    out.append(("zrl-past-se-first", grey(full + [scan((0,), 1, 10, 0, 0, [S(0x01), B(0, 1), ZRL]),
                                                 scan((0,), 11, 63, 0, 0, [S(0x22), B(2, 2), EOB])])))
    ref_pre = [scan((0,), 1, 63, 0, 1, [S(0x01), B(1, 1), S(0x21), B(0, 1), EOB])]   # zz1 = 2, zz4 = -2
    out.append(("zrl-eob-refine", grey(full + ref_pre + [scan((0,), 1, 63, 1, 0, [ZRL, B(1, 1), B(1, 1), EOB])])))
    out.append(("zrl-past-se-refine", grey(full + ref_pre + [scan((0,), 1, 10, 1, 0, [ZRL, B(0, 1), B(1, 1)]),
                                                            scan((0,), 11, 63, 1, 0, [EOB])])))
    # refinement symbols of every size 2..15 (only a warning in libjpeg): each still adds one +-1
    for s in (2, 7, 15):
        out.append((f"refine-size{s}", grey(full + [scan((0,), 1, 63, 0, 1, [EOB]),
                                                    scan((0,), 1, 63, 1, 0, [S(0x10 | s), B(1, 1), S(0x00 | s), B(0, 1), EOB])])))
    # EOB runs of 32767 in both AC scan kinds, over a 3x5 grey image (longer than the scan)
    run = [S(0xE0), B(0x3FFF, 14)]
    out.append(("eobrun-32767", grey([scan((0,), 0, 0, 0, 0, dc(1) + dc(-1) * 7 + dc(2) * 7), scan((0,), 1, 63, 0, 1, run),
                                      scan((0,), 1, 63, 1, 0, run)], blocks=(3, 5))))
    # an EOB run longer than the blocks left in its interval (restart 4 over 15 blocks): each interval resets it
    out.append(("eobrun-past-interval", grey([
        scan((0,), 0, 0, 0, 0, *[dc(k) + dc(0) * (3 if k < 4 else 2) for k in (1, 2, 3, 4)], restart=4),
        scan((0,), 1, 63, 0, 0, [S(0x01), B(1, 1), S(0x30), B(7, 3)], [S(0x40), B(3, 4)], [S(0x01), B(0, 1), S(0x20), B(2, 2)],
             [S(0x20), B(3, 2)], restart=4)], blocks=(3, 5))))
    # 16-bit codes: a table with one code of every length 1..16 (values placed on the longest codes)
    lengths = {0x00: 16, 0x01: 15, 0x02: 1, 0x11: 2, 0x12: 3, 0x21: 4, 0x22: 5, 0x31: 6, 0x32: 7, 0x41: 8, 0x42: 9, 0x51: 10,
               0x52: 11, 0x61: 12, 0x62: 13, 0x71: 14}
    out.append(("codes-16bit", grey(full + [scan((0,), 1, 63, 0, 0, [S(0x01), B(1, 1), S(0x01), B(0, 1), EOB],
                                                 huffman={0: J.table_from_lengths(lengths)})])))
    # one-symbol tables (the one code is "0") for DC and AC
    out.append(("one-symbol-tables", grey([scan((0,), 0, 0, 0, 0, [S(0)] * 3), scan((0,), 1, 63, 0, 0, [EOB] * 3)], blocks=(1, 3))))
    # a DHT redefined between two scans of one level: both use table 0 with other codes
    out.append(("dht-redefined-one-level", grey(full + [
        scan((0,), 1, 5, 0, 0, [S(0x01), B(1, 1), S(0x13), B(5, 3), EOB], huffman="optimal"),
        scan((0,), 21, 63, 0, 0, [S(0x42), B(1, 2), EOB]), scan((0,), 6, 20, 0, 0, [S(0x04), B(9, 4), EOB])])))
    # DC first at Al 13 with negative values, then its refinements
    out.append(("dc-al13-negative", grey([scan((0,), 0, 0, 0, 13, dc(-3) + dc(2) + dc(-1)), scan((0,), 1, 63, 0, 0, [S(0x20), B(2, 2)]),
                                          scan((0,), 0, 0, 13, 12, [B(0b101, 3)])], blocks=(1, 3))))
    # fill bytes (before markers and inside the data) and zero padding
    ff = [S(0x0E), B(0x3FFF, 14), EOB]                 # codes 00 / 01: bytes 7F FF 00, a stuffed 0xFF
    out.append(("fill-and-zero-pad", grey([
        scan((0,), 0, 0, 0, 0, dc(1), dc(-2), restart=1, fill=3, pad="zeros"),
        scan((0,), 1, 63, 0, 0, ff, ff, restart=1, fill=2, fill_data=2, pad="zeros")], blocks=(1, 2))))
    return out


def _dc_refine_cases() -> List[Tuple[str, bytes]]:
    """DC refinements over intervals that are not multiples of DC_REFINE_GROUP (16 blocks), jcphuff.c's own encoding."""
    rng = np.random.default_rng(3)
    blocks = np.zeros((5, 7, 8, 8), np.int64)
    blocks[..., 0, 0] = rng.integers(-300, 300, (5, 7))
    blocks[..., 0, 1] = rng.integers(-20, 20, (5, 7))
    script = [((0,), 0, 0, 0, 3), ((0,), 1, 63, 0, 0)] + [((0,), 0, 0, a + 1, a) for a in (2, 1, 0)]
    return [(f"dc-refine-restart{r}", W.write_progressive([blocks], {0: Q4}, height=40, width=56, sampling=[(1, 1)], script=script,
                                                          restart=r)) for r in (0, 1, 17, 20, 33)]


def exact_cases() -> List[Tuple[str, bytes]]:
    return _stray_cases() + _symbol_cases() + _dc_refine_cases()


# ---------------------------------------------------------------------------------------------------------------------
# Restart markers out of sequence
# ---------------------------------------------------------------------------------------------------------------------
def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([127.5 + 127.5 * np.sin(rng.uniform(0.02, 0.2) * (xx + yy * rng.uniform(0, 1)) + c) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 10, base.shape), 0, 255).astype(np.uint8)


def pil_file(img, **kw) -> bytes:
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=90, **kw)
    return b.getvalue()


def rst_markers(data: bytes) -> List[int]:
    """Offsets of the RSTn markers in the entropy-coded data of the first scan."""
    out, i = [], data.index(b"\xff\xda")
    i += 2 + int.from_bytes(data[i + 2:i + 4], "big")
    while i + 1 < len(data):
        if data[i] != 0xFF:
            i += 1
        elif data[i + 1] == 0xFF:    # a fill byte
            i += 1
        elif data[i + 1] == 0x00:
            i += 2
        elif 0xD0 <= data[i + 1] <= 0xD7:
            out.append(i)
            i += 2
        else:                        # the marker after the scan
            break
    return out


def renumbered(data: bytes, k: int, delta: int) -> bytes:
    at = rst_markers(data)[k]
    d = bytearray(data)
    d[at + 1] = 0xD0 + (d[at + 1] - 0xD0 + delta) % 8
    return bytes(d)


def dropped(data: bytes, k: int) -> bytes:
    at = rst_markers(data)[k]
    return data[:at] + data[at + 2:]


def added(data: bytes, k: int, num: int) -> bytes:
    """One more RSTn in the middle of the first scan's interval k (never between 0xFF and its stuffed 0x00)."""
    ms = rst_markers(data)
    sos = data.index(b"\xff\xda")
    start = ms[k - 1] + 2 if k else sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
    end = ms[k] if k < len(ms) else data.index(b"\xff", start + 1)
    mid = (start + end) // 2
    while data[mid - 1] == 0xFF or data[mid] == 0x00:
        mid += 1
    return data[:mid] + bytes([0xFF, 0xD0 + num]) + data[mid:]


def _resync_variants(f: bytes, plain: bytes) -> List[Tuple[str, bytes]]:
    out = [(f"rst{d:+d}", renumbered(f, 0, d)) for d in (1, 2, -1, -2, 4)]
    out += [("rst-mid+1", renumbered(f, 3, 1)), ("rst-missing", dropped(f, 1)), ("rst-missing-last", dropped(f, len(rst_markers(f)) - 1)),
            ("rst-extra", added(f, 2, 2)), ("rst-without-dri", added(plain, 0, 0))]
    return out


def resync_cases() -> List[Tuple[str, bytes]]:
    img = photo(32, 64, 0)
    return [("prog-" + n, d) for n, d in _resync_variants(pil_file(img, progressive=True, restart_marker_blocks=1),
                                                           pil_file(img, progressive=True))]


def baseline_resync_cases() -> List[Tuple[str, bytes]]:
    img = photo(32, 64, 0)
    out = [("base-" + n, d) for n, d in _resync_variants(pil_file(img, restart_marker_blocks=1), pil_file(img))]
    q = [J.quality_table(J.STD_Q_LUMA, 90), J.quality_table(J.STD_Q_CHROMA, 90)]
    coefs, samp = J.pixels_to_coefs(img, "420", q)
    w = J.write_jpeg(coefs, {0: q[0], 1: q[1]}, height=32, width=64, sampling=samp, restart=2, extra_rst=True)
    out.append(("base-extra-trailing", w.data))        # an in-sequence RSTn after the last interval: libjpeg ignores it
    return out
