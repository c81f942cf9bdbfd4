"""Video files in and out: ``open_video`` reads the frames of a video file, ``AviWriter`` writes Motion-JPEG AVI files.

Motion-JPEG in AVI is read by a RIFF parser of its own (``MjpegAvi``): every frame is a JPEG file, so it can take the same route
as a still image, to the GPU decoder when ``gpu_decodable`` says so, else to PIL on a host thread.  The frame chunks are found
through, in order of preference, the OpenDML (AVI 2.0) super index and its ``ix##`` chunks, the ``idx1`` index (offsets
relative to ``movi`` or absolute, whichever points at a chunk with the entry's id), or a walk over every ``movi`` list.  A
zero-length chunk is a dropped frame: it is skipped, and the other frames keep their index positions and so their times.  A
chunk payload is cut after the end of its first complete JPEG image: cameras pad their frames and some put a second field
behind the first, and PIL decodes the first image only.

Every other codec or container goes through OpenCV's FFmpeg backend (``FfmpegVideo``), decoded in order on the host.

``AviWriter`` writes RIFF ``AVI `` with one MJPG video stream, ``00dc`` chunks and an ``idx1`` in which every frame is a key
frame.  When the first RIFF would pass ``riff_limit`` bytes (1 GiB, the AVI 1.0 limit readers expect), the file continues in
OpenDML ``AVIX`` RIFFs, each ``movi`` list gets an ``ix00`` standard index, and the stream header gets an ``indx`` super index
and the file an ``odml``/``dmlh`` header.
"""
from __future__ import annotations

import os
import struct
import threading
from fractions import Fraction
from typing import Callable, Optional, Tuple

import numpy as np

# Codes MJPEG streams carry as their handler or biCompression, compared in upper case
MJPEG_FOURCCS = {b"MJPG", b"AVRN", b"DMB1", b"AVDJ", b"MJPA", b"JPGL", b"JPEG"}

AVIIF_KEYFRAME = 0x10
AVIF_HASINDEX = 0x10
AVI_INDEX_OF_INDEXES = 0x00
AVI_INDEX_OF_CHUNKS = 0x01
RIFF_LIMIT = 1 << 30


def sniff_video(head: bytes) -> bool:
    """True when the first bytes of a file are those of a video container: RIFF ``AVI ``, ISO-BMFF (``ftyp`` box, MP4 / MOV)
    or Matroska / WebM (EBML)."""
    return (head[:4] == b"RIFF" and head[8:12] == b"AVI ") or head[4:8] == b"ftyp" or head[:4] == b"\x1a\x45\xdf\xa3"


# ---------------------------------------------------------------------------------------------------------------------
# JPEG marker walk
# ---------------------------------------------------------------------------------------------------------------------
def jpeg_end(data) -> Optional[int]:
    """The offset just past the EOI marker of the first complete JPEG image in `data` (which starts with its SOI), or None when
    the data holds no complete image.  Walks the marker segments and skips each scan's entropy-coded data (stuffed zeros,
    fill bytes and RSTn belong to it)."""
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return None
    i = 2
    while True:
        while i < n and data[i] != 0xFF:
            i += 1
        while i < n and data[i] == 0xFF:
            i += 1
        if i >= n:
            return None
        m = data[i]
        i += 1
        if m == 0xD9:
            return i
        if 0xD0 <= m <= 0xD7 or m == 0x01 or m == 0xD8:
            continue
        if i + 2 > n:
            return None
        seg = (data[i] << 8) | data[i + 1]
        i += seg
        if m != 0xDA:
            continue
        while True:             # entropy-coded data: up to the next marker that is not RSTn
            j = data.find(b"\xff", i)
            if j < 0 or j + 1 >= n:
                return None
            b = data[j + 1]
            if b == 0xFF:
                i = j + 1
            elif b == 0x00 or 0xD0 <= b <= 0xD7:
                i = j + 2
            else:
                i = j
                break


def jpeg_hw(data) -> Tuple[int, int]:
    """(height, width) from the frame header of a JPEG file; ValueError when it has none."""
    n, i = len(data), 2
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise ValueError("not a JPEG file (no SOI marker)")
    while i + 4 <= n:
        if data[i] != 0xFF:
            i += 1
            continue
        m = data[i + 1]
        if m == 0xFF or 0xD0 <= m <= 0xD7 or m == 0x01:
            i += 1 if m == 0xFF else 2
            continue
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC) and i + 9 <= n:
            return (data[i + 5] << 8) | data[i + 6], (data[i + 7] << 8) | data[i + 8]
        if m in (0xD9, 0xDA):
            break
        i += 2 + ((data[i + 2] << 8) | data[i + 3])
    raise ValueError("JPEG file without a frame header")


def cut_frame(payload: bytes) -> bytes:
    """A Motion-JPEG chunk payload up to the end of its first complete JPEG image (the payload itself when it holds none)."""
    payload = bytes(payload)
    end = jpeg_end(payload)
    return payload if end is None else payload[:end]


# ---------------------------------------------------------------------------------------------------------------------
# Reading
# ---------------------------------------------------------------------------------------------------------------------
def _chunks(f, start: int, end: int):
    """(fourcc, data offset, size, list type or None) of the chunks between file offsets start and end; stops at a header that
    does not fit."""
    pos = start
    while pos + 8 <= end:
        f.seek(pos)
        hdr = f.read(12)
        if len(hdr) < 8:
            return
        cid, size = hdr[:4], struct.unpack("<I", hdr[4:8])[0]
        kind = hdr[8:12] if cid in (b"LIST", b"RIFF") and len(hdr) == 12 else None
        yield cid, pos + 8, size, kind
        pos += 8 + size + (size & 1)


class MjpegAvi:
    """The Motion-JPEG video stream of an AVI file, read by index.  Frames are numbered 0 .. n_frames - 1 in stream order,
    dropped (zero-length) chunks left out; ``position(k)`` is frame k's position in the stream, which gives its time."""

    def __init__(self, path: str):
        self.path = path
        self.size = os.path.getsize(path)
        with open(path, "rb") as f:
            self._parse(f)
        self.n_frames = len(self._entries)

    def _parse(self, f):
        f.seek(0)
        head = f.read(12)
        if not (head[:4] == b"RIFF" and head[8:12] == b"AVI "):
            raise ValueError(f"{self.path}: not an AVI file")
        riffs, hdrl, idx1 = [], None, None
        for cid, at, size, kind in _chunks(f, 0, self.size):
            if cid == b"RIFF" and kind in (b"AVI ", b"AVIX"):
                riffs.append((at, min(at + size, self.size)))
        for cid, at, size, kind in _chunks(f, riffs[0][0] + 4, riffs[0][1]):
            if cid == b"LIST" and kind == b"hdrl" and hdrl is None:
                hdrl = (at + 4, min(at + size, self.size))
            elif cid == b"idx1" and idx1 is None:
                idx1 = (at, min(size, self.size - at))
        if hdrl is None:
            raise ValueError(f"{self.path}: AVI file without a header list")
        self.movi = []      # offset of the 'movi' fourcc of each RIFF's movi list, and the list's end
        for r0, r1 in riffs:
            for cid, at, size, kind in _chunks(f, r0 + 4, r1):
                if cid == b"LIST" and kind == b"movi":
                    self.movi.append((at, min(at + size, self.size)))
        micro, stream, k = 0, None, 0
        for cid, at, size, kind in _chunks(f, *hdrl):
            if cid == b"avih" and size >= 4:
                f.seek(at)
                micro = struct.unpack("<I", f.read(4))[0]
            elif cid == b"LIST" and kind == b"strl":
                if stream is None:
                    stream = self._stream(f, at + 4, min(at + size, self.size), k)
                k += 1
        if stream is None:
            raise ValueError(f"{self.path}: no Motion-JPEG video stream")
        self.stream, handler, self._scale, self._rate, self.frame_hw, indx = stream
        self.codec = handler
        if self._rate == 0 and micro == 0:
            raise ValueError(f"{self.path}: the AVI gives no frame rate")
        self.fps = self._rate / self._scale if self._rate and self._scale else 1e6 / micro
        self._micro = micro
        ids = (b"%02ddc" % self.stream, b"%02ddb" % self.stream)
        self._ids = ids
        entries = (self._super_index(f, indx) if indx is not None else None)
        if entries is None and idx1 is not None:
            entries = self._idx1(f, *idx1)
        if entries is None:
            entries = self._scan(f)
        # (position in the stream, data offset, size) of every frame; zero-length chunks are dropped frames
        self._entries = [(p, at, n) for p, (at, n) in enumerate(entries) if n > 0]

    def _stream(self, f, start, end, k):
        strh = strf = indx = None
        for cid, at, size, kind in _chunks(f, start, end):
            f.seek(at)
            if cid == b"strh" and size >= 36:
                strh = f.read(min(size, 56))
            elif cid == b"strf" and size >= 20:
                strf = f.read(min(size, 40))
            elif cid == b"indx":
                indx = (at, size)
        if strh is None or strh[:4] != b"vids":
            return None
        handler, comp = strh[4:8], strf[16:20] if strf is not None else b""
        if handler.upper() not in MJPEG_FOURCCS and comp.upper() not in MJPEG_FOURCCS:
            return None
        scale, rate = struct.unpack("<II", strh[20:28])
        hw = (abs(struct.unpack("<i", strf[8:12])[0]), struct.unpack("<i", strf[4:8])[0]) if strf is not None else (0, 0)
        code = comp if comp.upper() in MJPEG_FOURCCS else handler
        return k, code.decode("latin-1"), scale, rate, hw, indx

    def _is_chunk(self, f, at, cid):
        if at < 0 or at + 8 > self.size:
            return False
        f.seek(at)
        hdr = f.read(8)
        return hdr[:4] == cid and at + 8 + struct.unpack("<I", hdr[4:8])[0] <= self.size

    def _idx1(self, f, at, size):
        f.seek(at)
        raw = np.frombuffer(f.read(size - size % 16), np.uint8).reshape(-1, 16)
        ids = raw[:, :4].tobytes()
        mine = [j for j in range(len(raw)) if ids[4 * j + 2:4 * j + 4] in (b"dc", b"db") and ids[4 * j:4 * j + 2] == self._ids[0][:2]]
        if not mine or not self.movi:
            return None
        offs = raw[:, 8:12].copy().view("<u4").reshape(-1).astype(np.int64)
        lens = raw[:, 12:16].copy().view("<u4").reshape(-1).astype(np.int64)
        j0 = mine[0]
        cid = ids[4 * j0:4 * j0 + 4]
        # most writers count from the 'movi' fourcc of the first movi list, some from the start of the file
        base = next((b for b in (self.movi[0][0], 0) if self._is_chunk(f, b + int(offs[j0]), cid)), None)
        if base is None:
            return None
        out = []
        for j in mine:
            at = base + int(offs[j]) + 8
            if at + int(lens[j]) > self.size:
                return None
            out.append((at, int(lens[j])))
        return out

    def _super_index(self, f, indx):
        at, size = indx
        f.seek(at)
        h = f.read(24)
        if len(h) < 24 or size < 24:
            return None
        per, _, kind, n = struct.unpack("<HBBI", h[:8])
        if kind != AVI_INDEX_OF_INDEXES or per != 4 or 24 + 16 * n > size:
            return None
        out = []
        for e in range(n):
            f.seek(at + 24 + 16 * e)
            qw, sz, _ = struct.unpack("<QII", f.read(16))
            if not self._is_chunk(f, qw, b"ix%02d" % self.stream):
                return None
            f.seek(qw + 8)
            ph = f.read(24)
            per_c, _, kind_c, m = struct.unpack("<HBBI", ph[:8])
            base = struct.unpack("<Q", ph[12:20])[0]
            if kind_c != AVI_INDEX_OF_CHUNKS or per_c != 2 or qw + 32 + 8 * m > self.size:
                return None
            raw = np.frombuffer(f.read(8 * m), "<u4").reshape(-1, 2).astype(np.int64)
            for off, ln in raw:
                ln = int(ln) & 0x7FFFFFFF
                if base + int(off) + ln > self.size:
                    return None
                out.append((base + int(off), ln))
        return out

    def _scan(self, f):
        out = []

        def walk(start, end):
            for cid, at, size, kind in _chunks(f, start, end):
                if cid == b"LIST" and kind == b"rec ":
                    walk(at + 4, min(at + size, end))
                elif cid in self._ids:
                    if at + size > self.size:
                        return False
                    out.append((at, size))
            return True

        for m0, m1 in self.movi:
            if not walk(m0 + 4, m1):
                break
        return out

    def position(self, k: int) -> int:
        return self._entries[k][0]

    def time(self, k: int) -> float:
        """Seconds from the start of the stream to frame k: its position * dwScale / dwRate (avih.dwMicroSecPerFrame when
        dwRate is 0)."""
        p = self._entries[k][0]
        return p * self._scale / self._rate if self._rate and self._scale else p * self._micro / 1e6

    def payload(self, k: int) -> bytes:
        """Frame k's chunk payload as stored."""
        _, at, n = self._entries[k]
        with open(self.path, "rb") as f:
            f.seek(at)
            return f.read(n)

    def frame_bytes(self, k: int) -> bytes:
        """Frame k: its chunk payload cut after the end of its first complete JPEG image."""
        return cut_frame(self.payload(k))

    def loader(self, keep: Optional[Callable[[int], bool]] = None, route: Optional[Callable] = None):
        """A function from a frame number to what ``DetectionPipeline.submit_images`` takes: ``route(frame bytes)`` (default:
        the bytes).  Safe to call from several threads in any order; `keep` is not needed (every frame is read by index)."""
        route = route or (lambda b: b)
        return lambda k: route(self.frame_bytes(k))

    def frames(self):
        for k in range(self.n_frames):
            yield self.frame_bytes(k)


class FfmpegVideo:
    """Any other video OpenCV's FFmpeg backend reads, decoded in stream order on the host: RGB uint8 [h, w, 3] frames, as
    that backend gives them (BGR turned to RGB)."""

    def __init__(self, path: str):
        import cv2
        cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
        if not cap.isOpened():
            raise ValueError(f"{path}: not a video file OpenCV's FFmpeg backend can read")
        self.path = path
        self.fps = float(cap.get(cv2.CAP_PROP_FPS))
        self.frame_hw = (int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)))
        four = int(cap.get(cv2.CAP_PROP_FOURCC))
        self.codec = bytes((four >> s) & 255 for s in (0, 8, 16, 24)).decode("latin-1")
        n = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        if n <= 0:          # the container gives no count: one pass over the stream counts the frames
            n = 0
            while cap.grab():
                n += 1
        cap.release()
        self.n_frames = n
        if self.fps <= 0:
            raise ValueError(f"{path}: the video gives no frame rate")

    def position(self, k: int) -> int:
        return k

    def time(self, k: int) -> float:
        return k / self.fps

    def loader(self, keep: Optional[Callable[[int], bool]] = None, route: Optional[Callable] = None):
        """A function from a frame number to its RGB pixels.  The stream is decoded once, in order, behind a lock, whatever
        order the calls come in; frames for which `keep` is true (default: all) are held until they are asked for, the others
        are decoded and dropped."""
        import cv2
        cap = cv2.VideoCapture(self.path, cv2.CAP_FFMPEG)
        if not cap.isOpened():
            raise ValueError(f"{self.path}: cannot open")
        lock, held, state = threading.Lock(), {}, {"next": 0}
        keep = keep or (lambda k: True)

        def load(k):
            with lock:
                while k not in held and state["next"] <= k:
                    j = state["next"]
                    ok, bgr = cap.read()
                    if not ok:
                        raise ValueError(f"{self.path}: the stream ends at frame {j} of {self.n_frames}")
                    state["next"] += 1
                    if keep(j):
                        held[j] = np.ascontiguousarray(bgr[..., ::-1])
                if k not in held:
                    raise ValueError(f"{self.path}: frame {k} was asked for after the stream passed it")
                return held.pop(k)

        return load

    def frames(self):
        load = self.loader()
        for k in range(self.n_frames):
            yield load(k)


def open_video(path: str):
    """The video stream of a file: ``MjpegAvi`` for an AVI with a Motion-JPEG video stream, ``FfmpegVideo`` for anything
    else.  Either exposes ``n_frames``, ``fps``, ``frame_hw``, ``codec``, ``time(k)``, ``position(k)``, ``frames()`` and
    ``loader(keep, route)``."""
    with open(path, "rb") as f:
        head = f.read(12)
    if head[:4] == b"RIFF" and head[8:12] == b"AVI ":
        try:
            return MjpegAvi(path)
        except ValueError as e:
            if "no Motion-JPEG video stream" not in str(e):
                raise
    return FfmpegVideo(path)


# ---------------------------------------------------------------------------------------------------------------------
# Writing
# ---------------------------------------------------------------------------------------------------------------------
_DMLH_BYTES = 248


class AviWriter:
    """Writes JPEG files one frame at a time as a Motion-JPEG AVI of `fps` frames per second and frame size `hw` (h, w).
    Past `riff_limit` bytes in the first RIFF the file continues as OpenDML (AVI 2.0); `max_riffs` bounds the RIFFs the
    super index has room for.  Use as a context manager, or call ``close``."""

    def __init__(self, path: str, fps, hw, riff_limit: int = RIFF_LIMIT, max_riffs: int = 1024):
        self.path, self.hw = path, (int(hw[0]), int(hw[1]))
        r = Fraction(fps).limit_denominator(1_000_000)
        if r <= 0:
            raise ValueError(f"frame rate {fps} is not positive")
        self.rate, self.scale = r.numerator, r.denominator
        self.limit, self.max_riffs = int(riff_limit), int(max_riffs)
        self.f = open(path, "wb")
        self.n = 0
        self.max_chunk = 0
        self.riffs = []         # per RIFF: [riff offset, movi offset, [(data offset, size)], ix00 offset]
        self._header()
        self._start_riff(b"AVI ")

    def _u32(self, v):
        return struct.pack("<I", v & 0xFFFFFFFF)

    def _header(self):
        f = self.f
        f.write(b"RIFF" + bytes(4) + b"AVI ")
        self._hdrl = f.tell()
        f.write(b"LIST" + bytes(4) + b"hdrl")
        self._avih = f.tell()
        f.write(b"avih" + self._u32(56) + bytes(56))
        strl = f.tell()
        f.write(b"LIST" + bytes(4) + b"strl")
        self._strh = f.tell()
        f.write(b"strh" + self._u32(56) + bytes(56))
        h, w = self.hw
        f.write(b"strf" + self._u32(40) + struct.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, b"MJPG", w * h * 3, 0, 0, 0, 0))
        self._indx = f.tell()      # room for the super index, a JUNK chunk until the file needs one
        self._indx_bytes = 24 + 16 * self.max_riffs
        f.write(b"JUNK" + self._u32(self._indx_bytes) + bytes(self._indx_bytes))
        self._patch(strl + 4, f.tell() - strl - 8)
        self._odml = f.tell()      # room for LIST odml / dmlh
        f.write(b"JUNK" + self._u32(12 + _DMLH_BYTES) + bytes(12 + _DMLH_BYTES))
        self._patch(self._hdrl + 4, f.tell() - self._hdrl - 8)

    def _patch(self, at, value, fmt="<I"):
        here = self.f.tell()
        self.f.seek(at)
        self.f.write(struct.pack(fmt, value))
        self.f.seek(here)

    def _start_riff(self, kind):
        f = self.f
        riff = 0 if kind == b"AVI " else f.tell()
        if kind != b"AVI ":
            f.write(b"RIFF" + bytes(4) + kind)
        movi = f.tell()
        f.write(b"LIST" + bytes(4) + b"movi")
        self.riffs.append([riff, movi, [], None])

    def _index_bytes(self, frames):
        first = len(self.riffs) == 1
        return (8 + 16 * frames if first else 0) + 32 + 8 * frames

    def write(self, jpeg: bytes) -> None:
        """Appends one frame (the bytes of a JPEG file).  ValueError when its size is not the stream's."""
        hw = jpeg_hw(jpeg)
        if hw != self.hw:
            raise ValueError(f"{self.path}: frame {self.n} is {hw[1]}x{hw[0]}, the stream is {self.hw[1]}x{self.hw[0]}: "
                             "an AVI stream has one frame size")
        f = self.f
        size = len(jpeg)
        riff = self.riffs[-1]
        used = f.tell() - riff[0] + 8 + size + (size & 1) + self._index_bytes(len(riff[2]) + 1)
        if riff[2] and used > self.limit:
            self._end_riff(opendml=True)
            if len(self.riffs) == self.max_riffs:
                raise ValueError(f"{self.path}: more than {self.max_riffs} RIFFs")
            self._start_riff(b"AVIX")
            riff = self.riffs[-1]
        f.write(b"00dc" + self._u32(size))
        riff[2].append((f.tell(), size))
        f.write(jpeg)
        if size & 1:
            f.write(b"\0")
        self.n += 1
        self.max_chunk = max(self.max_chunk, size)

    def _end_riff(self, opendml):
        """Closes the last RIFF: its ix00 when the file is OpenDML, the movi size, the idx1 of the first RIFF, the RIFF size."""
        f = self.f
        riff, movi, entries, _ = self.riffs[-1]
        if opendml:
            self.riffs[-1][3] = f.tell()
            base = movi + 8
            f.write(b"ix00" + self._u32(24 + 8 * len(entries)) + struct.pack("<HBBI4sQI", 2, 0, AVI_INDEX_OF_CHUNKS, len(entries),
                                                                              b"00dc", base, 0))
            f.write(b"".join(struct.pack("<II", at - base, n) for at, n in entries))
        self._patch(movi + 4, f.tell() - movi - 8)
        if len(self.riffs) == 1:
            f.write(b"idx1" + self._u32(16 * len(entries)))
            f.write(b"".join(struct.pack("<4sIII", b"00dc", AVIIF_KEYFRAME, at - 8 - (movi + 8), n) for at, n in entries))
        self._patch(riff + 4, f.tell() - riff - 8)

    def close(self) -> None:
        if self.f is None:
            return
        f = self.f
        opendml = len(self.riffs) > 1
        self._end_riff(opendml)
        first = len(self.riffs[0][2])
        h, w = self.hw
        us = round(1e6 * self.scale / self.rate)
        f.seek(self._avih + 8)
        f.write(struct.pack("<IIIIIIIIII16x", us, 0, 0, AVIF_HASINDEX, first, 0, 1, self.max_chunk, w, h))
        f.seek(self._strh + 8)
        f.write(struct.pack("<4s4sIHHIIIIIIIIhhhh", b"vids", b"MJPG", 0, 0, 0, 0, self.scale, self.rate, 0, self.n,
                            self.max_chunk, 0xFFFFFFFF, 0, 0, 0, w, h))
        if opendml:
            f.seek(self._indx)
            f.write(b"indx" + self._u32(self._indx_bytes) + struct.pack("<HBBI4s12x", 4, 0, AVI_INDEX_OF_INDEXES, len(self.riffs), b"00dc"))
            for _, _, entries, ix in self.riffs:
                f.write(struct.pack("<QII", ix, 32 + 8 * len(entries), len(entries)))
            f.seek(self._odml)
            f.write(b"LIST" + self._u32(4 + 8 + _DMLH_BYTES) + b"odml" + b"dmlh" + self._u32(_DMLH_BYTES) + self._u32(self.n))
        f.close()
        self.f = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
