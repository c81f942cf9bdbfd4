"""PNG files for the decoder tests, written chunk by chunk: any colour type and depth, rows filtered by the test (each row its
own filter type), the zlib stream from zlib at any level and strategy or from oracle/deflate_ref.py, split over IDATs anywhere."""
from __future__ import annotations

import io
import struct
import zlib
from typing import Optional, Sequence

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
GPU_KINDS = [(0, 1), (0, 2), (0, 4), (0, 8), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16), (6, 8), (6, 16)]


def chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def ihdr(w: int, h: int, color: int, depth: int, interlace: int = 0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color, 0, 0, interlace))


def row_bytes(w: int, color: int, depth: int) -> int:
    return (w * CHANNELS[color] * depth + 7) // 8


def random_rows(rng, w: int, h: int, color: int, depth: int, content: str = "noise", plte_n: int = 256) -> np.ndarray:
    """Unfiltered rows, uint8 [h, rowbytes]: "noise", "flat", "photo" (smooth gradients + noise) or "detail" (sharp edges)."""
    rb = row_bytes(w, color, depth)
    if content == "flat":
        rows = np.full((h, rb), rng.integers(0, 256), np.uint8)
    elif content == "photo":
        base = (np.add.outer(np.arange(h), np.arange(rb) // max(1, CHANNELS[color] * depth // 8)) * 3) % 256
        rows = (base + rng.integers(0, 6, (h, rb))).astype(np.uint8)
    elif content == "detail":
        rows = (((np.arange(h)[:, None] // 3 + np.arange(rb)[None, :] // 5) % 2) * 255).astype(np.uint8)
        rows ^= rng.integers(0, 2, (h, rb)).astype(np.uint8)
    else:
        rows = rng.integers(0, 256, (h, rb), dtype=np.uint8)
    if color == 3 and depth == 8:
        rows = (rows.astype(np.int64) % max(1, plte_n + 2)).astype(np.uint8)     # a few indices past the PLTE entries
    pad = rb * 8 - w * CHANNELS[color] * depth
    if pad:
        rows[:, -1] &= np.uint8((0xFF << pad) & 0xFF) if rng.integers(0, 2) else np.uint8(0xFF)   # padding bits: zero or not
    return rows


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows: np.ndarray, bpp: int, types: Sequence[int]) -> bytes:
    """The filtered scanlines (type byte + row) of unfiltered `rows` with filter types[r % len(types)] on row r."""
    out = bytearray()
    prev = np.zeros(rows.shape[1], np.int64)
    for r in range(rows.shape[0]):
        cur = rows[r].astype(np.int64)
        left = np.concatenate([np.zeros(bpp, np.int64), cur[:-bpp]])[:len(cur)]
        upleft = np.concatenate([np.zeros(bpp, np.int64), prev[:-bpp]])[:len(cur)]
        t = types[r % len(types)]
        pred = [0, left, prev, (left + prev) // 2, _paeth(left, prev, upleft)][t]
        out.append(t)
        out += ((cur - pred) % 256).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def bpp_of(color: int, depth: int) -> int:
    return max(1, CHANNELS[color] * depth // 8)


def png_file(w: int, h: int, color: int, depth: int, stream: bytes, plte: Optional[bytes] = None, split: Optional[Sequence[int]] = None,
             before: bytes = b"", between: bytes = b"", after: bytes = b"", iend: bool = True, interlace: int = 0) -> bytes:
    """A PNG with zlib `stream` cut into IDATs at the byte offsets `split` (repeats give empty IDATs); `before` goes after
    IHDR/PLTE, `between` after the first IDAT and `after` after the last."""
    cuts = [0] + sorted(split or []) + [len(stream)]
    idats = [chunk(b"IDAT", stream[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    body = idats[0] + between + b"".join(idats[1:])
    out = SIG + ihdr(w, h, color, depth, interlace) + (chunk(b"PLTE", plte) if plte is not None else b"") + before + body + after
    return out + (chunk(b"IEND", b"") if iend else b"")


def make_png(rng, w: int, h: int, color: int, depth: int, content: str = "noise", types: Sequence[int] = (0, 1, 2, 3, 4),
             level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY, plte_n: int = 200, split=None) -> bytes:
    """A whole file: random rows, filtered with `types` in turn, compressed by zlib at `level` with `strategy`."""
    plte = rng.integers(0, 256, 3 * plte_n, dtype=np.uint8).tobytes() if color == 3 else None
    rows = random_rows(rng, w, h, color, depth, content, plte_n)
    raw = filter_rows(rows, bpp_of(color, depth), types)
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    return png_file(w, h, color, depth, co.compress(raw) + co.flush(), plte, split)


def pil_png(img: np.ndarray, **kw) -> bytes:
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "PNG", **kw)
    return b.getvalue()


def pil_read(data: bytes):
    """``read_image`` of the file, or the exception PIL raises."""
    from k210_yolo_framework_b200.helper import read_image
    try:
        return read_image(io.BytesIO(data))
    except Exception as e:      # PIL raises several types for damaged files
        return e
