"""Detection results drawn and JPEG-encoded on the GPU, with the bytes the host route (``draw.draw_detections`` + PIL ``save``)
gives.

``render_detections_device`` draws a batch of records onto CUDA uint8 [h, w, 3] images in place, in one launch
(``k2y_render_detections``, csrc/render.cu): the outline rings, the filled label box and the black label text of every record,
pixel for pixel what ``draw.draw_detections`` draws.  The label glyphs come from a ``LabelAtlas``: per font, the 8-bit mask,
mask offset and ``textbbox`` size of every ``(class, hundredths)`` label, taken from Pillow on the host exactly as
``ImageDraw.text`` / ``textbbox`` get them, cached per font size and uploaded once.

``render_tracks_device`` draws a tracker's output the same way (``k2y_render_tracks``), as ``draw.draw_tracks`` draws it:
each record's track box in its id's colour, labelled ``"{class:2d} #{id}"``.  Ids are unbounded, so its ``TrackLabelAtlas``
holds the label's 12 glyphs per font size and the kernel composes each label from them.

``encode_jpeg_batch`` encodes CUDA uint8 [h, w, 3] images as baseline JPEG files byte-identical to
``PIL.Image.fromarray(x).save(f, "JPEG", quality=q)`` (``k2y_jpeg_encode``, csrc/jpeg_encode.cu): the headers are built on the
host, colour conversion, downsampling, FDCT, quantisation, Huffman coding and byte stuffing run on the device, one launch per
stage for the whole batch, and only the compressed files come back.  ``JpegEncoder`` is the reusable form the pipeline uses.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ._lib import K2YError, check, lib
from .draw import label_font_size

LABELS_PER_CLASS = 101      # hundredths 0..100
HEADER_WORDS = 8            # atlas header: [0] classes
ENTRY_WORDS = 8             # mask byte offset, mask w, mask h, mask x, mask y, label w, label h, 0
MAX_CLASSES = 80            # the colour table's classes (Helper.colormap)
TRACK_GLYPHS = "0123456789 #"   # the glyphs of a track label, in track atlas order
TRACK_ENTRY_WORDS = 10      # mask byte offset, mask w, mask h, mask x, mask y, textbbox left, top, right, bottom, advance
JPEG_MAX_DIMENSION = 65500  # libjpeg-turbo's limit: PIL neither writes nor reads a JPEG with more rows or columns
_LL = ctypes.POINTER(ctypes.c_longlong)
_INT = ctypes.POINTER(ctypes.c_int)


def label_text(cls: int, hundredths: int) -> str:
    """``"{:2d} {:.2f}".format(cls, score)`` for a score that rounds to `hundredths` / 100."""
    return "{:2d} {}.{:02d}".format(int(cls), hundredths // 100, hundredths % 100)


def label_hundredths(score: float) -> int:
    """The hundredths ``"{:.2f}"`` prints for a float32 score: rint(double(score) * 100), exact and ties to even."""
    return int(np.rint(np.float64(np.float32(score)) * 100.0))


def glyphs(font, label: str):
    """(mask uint8 [mh, mw], (mask x, mask y), (label w, label h)) of `label` as ``ImageDraw.text`` draws it at an integer origin
    on an RGB image, and the size ``ImageDraw.textbbox`` gives."""
    from PIL import Image, ImageDraw
    draw = ImageDraw.Draw(Image.new("RGB", (1, 1)))
    tb = draw.textbbox((0, 0), label, font=font)
    try:
        mask, offset = font.getmask2(label, draw.fontmode, anchor="la", ink=0, start=(0.0, 0.0))
    except AttributeError:      # a bitmap font without getmask2: ImageDraw.text falls back to getmask at the origin
        mask, offset = font.getmask(label, draw.fontmode), (0, 0)
    mw, mh = mask.size
    arr = np.array(mask, dtype=np.uint8).reshape(mh, mw) if mw * mh else np.zeros((mh, mw), np.uint8)
    return arr, (int(offset[0]), int(offset[1])), (int(tb[2] - tb[0]), int(tb[3] - tb[1]))


def build_atlas(font, class_num: int) -> np.ndarray:
    """The atlas words of `font` for classes 0..class_num-1: int32 header [8], entries [class_num][101][8], then the masks."""
    entries = np.zeros((class_num * LABELS_PER_CLASS, ENTRY_WORDS), np.int32)
    masks, off = [], 0
    for c in range(class_num):
        for h in range(LABELS_PER_CLASS):
            m, (mx, my), (lw, lh) = glyphs(font, label_text(c, h))
            entries[c * LABELS_PER_CLASS + h] = (off, m.shape[1], m.shape[0], mx, my, lw, lh, 0)
            masks.append(m.reshape(-1))
            off += m.size
    blob = np.concatenate(masks + [np.zeros((-off) % 4, np.uint8)]) if masks else np.zeros(0, np.uint8)
    header = np.zeros(HEADER_WORDS, np.int32)
    header[0] = class_num
    return np.concatenate([header, entries.reshape(-1), blob.view(np.int32)])


class _FontAtlas:
    """Atlas words per font size of the font ``draw.label_font`` picks per image height, built on the host once per size
    (``_build(font)``) and uploaded once per device."""

    def __init__(self, font_path: str):
        self.font_path = font_path
        self._key_of_size: Dict[int, object] = {}
        self._host: Dict[object, np.ndarray] = {}
        self._dev: Dict[tuple, torch.Tensor] = {}

    def _key(self, image_h: int):
        size = label_font_size(image_h)
        key = self._key_of_size.get(size)
        if key is None:
            from PIL import ImageFont
            try:
                font = ImageFont.truetype(font=self.font_path, size=size)
                key = ("truetype", size)
            except (OSError, ValueError):    # ValueError: size 0 below 17 rows, where draw_detections raises instead
                font = ImageFont.load_default()
                key = ("default",)
            if key not in self._host:
                self._host[key] = self._build(font)
            self._key_of_size[size] = key
        return key

    def host(self, image_h: int) -> np.ndarray:
        return self._host[self._key(image_h)]

    def device(self, image_h: int, device: torch.device) -> torch.Tensor:
        key = (self._key(image_h), device)
        t = self._dev.get(key)
        if t is None:
            t = torch.from_numpy(self._host[key[0]]).to(device)
            torch.cuda.synchronize(device)      # visible to every stream before first use
            self._dev[key] = t
        return t


class LabelAtlas(_FontAtlas):
    """The label glyphs of every ``(class, hundredths)`` for the font ``draw.label_font`` picks per image height, built on the
    host once per font size (about 0.3 s per 2020 labels) and uploaded once per device."""

    def __init__(self, class_num: int, font_path: str = "asset/FiraMono-Medium.otf"):
        if not 1 <= int(class_num) <= MAX_CLASSES:
            raise ValueError(f"class_num {class_num} is outside 1..{MAX_CLASSES}")
        super().__init__(font_path)
        self.class_num = int(class_num)

    def _build(self, font) -> np.ndarray:
        return build_atlas(font, self.class_num)


def check_track_font(font) -> None:
    """Raises ``ValueError`` unless the advances of the track label's glyphs are whole pixels that add up without kerning,
    over every pair: then glyph i of a label starts at the integer pen position sum(advance[c_j] for j < i), which is what
    ``k2y_render_tracks`` composes the label from."""
    adv = {}
    for ch in TRACK_GLYPHS:
        a = font.getlength(ch)
        if a != int(a):
            raise ValueError(f"the advance of {ch!r} is {a} pixels, not a whole number: track labels cannot be composed per glyph")
        adv[ch] = int(a)
    for a in TRACK_GLYPHS:
        for b in TRACK_GLYPHS:
            if font.getlength(a + b) != adv[a] + adv[b]:
                raise ValueError(f"{a + b!r} advances {font.getlength(a + b)} pixels, not {adv[a]} + {adv[b]} (kerning): track "
                                 "labels cannot be composed per glyph")


def build_track_atlas(font) -> np.ndarray:
    """The track atlas words of `font`: int32 header [8] ([0] glyphs), entries [12][10] of the glyphs of ``TRACK_GLYPHS``
    (mask byte offset, mask w, mask h, mask x, mask y, textbbox left, top, right, bottom, advance), then the masks.  Raises
    ``ValueError`` for a font ``check_track_font`` refuses."""
    from PIL import Image, ImageDraw
    check_track_font(font)
    draw = ImageDraw.Draw(Image.new("RGB", (1, 1)))
    entries = np.zeros((len(TRACK_GLYPHS), TRACK_ENTRY_WORDS), np.int32)
    masks, off = [], 0
    for g, ch in enumerate(TRACK_GLYPHS):
        m, (mx, my), _ = glyphs(font, ch)
        tb = draw.textbbox((0, 0), ch, font=font)
        entries[g] = (off, m.shape[1], m.shape[0], mx, my, tb[0], tb[1], tb[2], tb[3], int(font.getlength(ch)))
        masks.append(m.reshape(-1))
        off += m.size
    blob = np.concatenate(masks + [np.zeros((-off) % 4, np.uint8)])
    header = np.zeros(HEADER_WORDS, np.int32)
    header[0] = len(TRACK_GLYPHS)
    return np.concatenate([header, entries.reshape(-1), blob.view(np.int32)])


class TrackLabelAtlas(_FontAtlas):
    """The 12 glyphs of the track labels ``"{class:2d} #{track_id}"`` (``TRACK_GLYPHS``: digits, space and ``#``) for the
    font ``draw.label_font`` picks per image height: per glyph the mask and mask offset ``ImageDraw.text`` draws it with, its
    ``textbbox`` and its advance, built on the host once per font size and uploaded once per device.  ``k2y_render_tracks``
    composes any label from them, ids being unbounded.  Raises ``ValueError`` (when a font size is first used) for a font
    whose advances of these glyphs are fractional or kern."""

    def __init__(self, font_path: str = "asset/FiraMono-Medium.otf"):
        super().__init__(font_path)

    @staticmethod
    def _build(font) -> np.ndarray:
        return build_track_atlas(font)


def color_table(colormap, class_num: int, device: torch.device) -> torch.Tensor:
    if class_num > len(colormap):
        raise ValueError(f"class_num {class_num} exceeds the colormap's {len(colormap)} entries")
    t = torch.tensor(np.asarray(colormap[:class_num], np.uint8).reshape(class_num, 3)).to(device)
    torch.cuda.synchronize(device)
    return t


def _check_views(images: Sequence[torch.Tensor]):
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("expected a non-empty list of CUDA uint8 [h, w, 3] tensors")
    dev = images[0].device
    for i, t in enumerate(images):
        if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3
                or not t.is_contiguous() or t.device != dev):
            raise ValueError(f"image {i}: expected a contiguous CUDA uint8 [h, w, 3] tensor on {dev}")
        if not (1 <= t.shape[0] <= 65535 and 1 <= t.shape[1] <= 65535):
            raise ValueError(f"image {i} is {t.shape[0]}x{t.shape[1]}; 1..65535 rows and columns are supported")
    base = min(t.data_ptr() for t in images)
    offsets = np.array([t.data_ptr() - base for t in images], np.int64)
    hw = np.array([[t.shape[0], t.shape[1]] for t in images], np.int32)
    return dev, base, offsets, hw


def render_packed(base_ptr: int, offsets: np.ndarray, hw: np.ndarray, dets: torch.Tensor, counts: torch.Tensor, atlas: LabelAtlas,
                  colors: torch.Tensor, device: torch.device, stream: torch.cuda.Stream) -> None:
    """``k2y_render_detections`` over images packed at `offsets` from `base_ptr` (device), asynchronous on `stream`."""
    n = len(offsets)
    C, K = atlas.class_num, dets.shape[2]
    if (dets.dtype != torch.int32 or counts.dtype != torch.int32 or dets.dim() != 4 or tuple(dets.shape[1:]) != (C, K, 6) or
            tuple(dets.stride()[1:]) != (K * 6, 6, 1) or counts.dim() != 2 or counts.shape[1] != C or counts.stride(1) != 1 or
            dets.shape[0] < n or counts.shape[0] < n or not dets.is_cuda or not counts.is_cuda):
        raise ValueError(f"dets must be CUDA int32 [n, {C}, K, 6] dense per image, counts CUDA int32 [n, {C}]")
    tables = [atlas.device(int(h), device) for h, _ in hw]
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tables])
    offsets = np.ascontiguousarray(offsets, np.int64)
    hw = np.ascontiguousarray(hw, np.int32)
    check(lib.k2y_render_detections(ctypes.c_void_p(base_ptr), n, offsets.ctypes.data_as(_LL), hw.ctypes.data_as(_INT), ptrs,
                                    dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0), C, K, colors.data_ptr(),
                                    ctypes.c_void_p(stream.cuda_stream)))


def render_detections_device(images: Sequence[torch.Tensor], dets: torch.Tensor, counts: torch.Tensor, atlas: LabelAtlas,
                             colormap=None, stream: Optional[torch.cuda.Stream] = None) -> None:
    """Draws image i's records (``dets[i]`` int32 [C, K, 6] k2y_det words, ``counts[i]`` [C], device tensors as the detector or
    a gather buffer holds them) onto ``images[i]`` (contiguous CUDA uint8 [h, w, 3]) in place, as ``draw.draw_detections``
    would; asynchronous on `stream` (default: the current stream).  `colormap`: RGB triples per class (default
    ``Helper.colormap``)."""
    from .helper import _COLORMAP
    dev, base, offsets, hw = _check_views(images)
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    colors = color_table(_COLORMAP if colormap is None else colormap, atlas.class_num, dev)
    with torch.cuda.device(dev):
        render_packed(base, offsets, hw, dets, counts, atlas, colors, dev, st)
    colors.record_stream(st)


def track_color_table(colormap, device: torch.device) -> torch.Tensor:
    """Every colormap entry on the device: a track's colour is ``colormap[id % len(colormap)]``."""
    if len(colormap) < 1:
        raise ValueError("the colormap has no colours")
    t = torch.tensor(np.asarray(colormap, np.uint8).reshape(len(colormap), 3)).to(device)
    torch.cuda.synchronize(device)
    return t


def render_tracks_packed(base_ptr: int, offsets: np.ndarray, hw: np.ndarray, counts: torch.Tensor, ids: torch.Tensor,
                         boxes: torch.Tensor, atlas: TrackLabelAtlas, colors: torch.Tensor, device: torch.device,
                         stream: torch.cuda.Stream) -> None:
    """``k2y_render_tracks`` over images packed at `offsets` from `base_ptr` (device), asynchronous on `stream`."""
    n = len(offsets)
    if ids.dim() != 3 or counts.dim() != 2:
        raise ValueError("ids must be CUDA int32 [n, C, K], boxes CUDA float32 [n, C, K, 4], counts CUDA int32 [n, C]")
    C, K = ids.shape[1], ids.shape[2]
    if (ids.dtype != torch.int32 or boxes.dtype != torch.float32 or counts.dtype != torch.int32 or
            tuple(ids.stride()[1:]) != (K, 1) or boxes.dim() != 4 or tuple(boxes.shape[1:]) != (C, K, 4) or
            tuple(boxes.stride()[1:]) != (K * 4, 4, 1) or counts.shape[1] != C or counts.stride(1) != 1 or
            min(ids.shape[0], boxes.shape[0], counts.shape[0]) < n or not (ids.is_cuda and boxes.is_cuda and counts.is_cuda)):
        raise ValueError(f"ids must be CUDA int32 [n, C, K], boxes CUDA float32 [n, C, K, 4], counts CUDA int32 [n, C], dense per "
                         f"image (got {tuple(ids.shape)}, {tuple(boxes.shape)}, {tuple(counts.shape)})")
    if not 1 <= C <= MAX_CLASSES:
        raise ValueError(f"class_num {C} is outside 1..{MAX_CLASSES}")
    tables = [atlas.device(int(h), device) for h, _ in hw]
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tables])
    offsets = np.ascontiguousarray(offsets, np.int64)
    hw = np.ascontiguousarray(hw, np.int32)
    check(lib.k2y_render_tracks(ctypes.c_void_p(base_ptr), n, offsets.ctypes.data_as(_LL), hw.ctypes.data_as(_INT), ptrs,
                                ids.data_ptr(), boxes.data_ptr(), counts.data_ptr(), ids.stride(0), boxes.stride(0), counts.stride(0),
                                C, K, colors.data_ptr(), colors.shape[0], ctypes.c_void_p(stream.cuda_stream)))


def render_tracks_device(images: Sequence[torch.Tensor], counts: torch.Tensor, ids: torch.Tensor, boxes: torch.Tensor,
                         atlas: TrackLabelAtlas, colormap=None, stream: Optional[torch.cuda.Stream] = None) -> None:
    """Draws image i's tracks onto ``images[i]`` (contiguous CUDA uint8 [h, w, 3]) in place, as ``draw.draw_tracks`` would:
    record k of class c (k < ``counts[i, c]``, int32 [n, C]) with ``ids[i, c, k]`` >= 0 (int32 [n, C, K]) is drawn with its
    track box ``boxes[i, c, k]`` (float32 [n, C, K, 4], ymin, xmin, ymax, xmax), labelled ``"{c:2d} #{id}"``, in colour
    ``colormap[id % len(colormap)]`` (default ``Helper.colormap``): the layout ``DetectionPipeline.tracks`` returns, as device
    tensors.  Asynchronous on `stream` (default: the current stream)."""
    from .helper import _COLORMAP
    dev, base, offsets, hw = _check_views(images)
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    colors = track_color_table(_COLORMAP if colormap is None else colormap, dev)
    with torch.cuda.device(dev):
        render_tracks_packed(base, offsets, hw, counts, ids, boxes, atlas, colors, dev, st)
    colors.record_stream(st)


class JpegEncoder:
    """Reusable buffers of ``k2y_jpeg_encode``: a pinned blob, its device copy, the workspace, the packed output and the
    lengths (device and pinned host).  ``enqueue`` encodes a batch asynchronously; once the stream has passed it
    (``ready`` event synchronised), ``fetch`` returns the files with one exact-size device-to-host copy."""

    def __init__(self, device: torch.device):
        self.device = device
        self._blob_host: Optional[torch.Tensor] = None
        self._blob_dev: Optional[torch.Tensor] = None
        self._ws: Optional[torch.Tensor] = None
        self.out: Optional[torch.Tensor] = None
        self._len_dev: Optional[torch.Tensor] = None
        self.lengths_host: Optional[torch.Tensor] = None
        self.n = 0
        self.ready = torch.cuda.Event()

    @staticmethod
    def _grow(t: Optional[torch.Tensor], n: int, **kw) -> torch.Tensor:
        if t is not None and t.numel() >= n:
            return t
        return torch.empty((max(n, 2 * t.numel() if t is not None else 0),), **kw)

    def enqueue(self, base_ptr: int, offsets: np.ndarray, hw: np.ndarray, quality: int, stream: torch.cuda.Stream) -> None:
        """Encodes the images packed at `offsets` from `base_ptr` (int64 [n], hw int32 [n, 2]) on `stream`.  The previous
        batch's files are lost: fetch them first."""
        q = int(quality)
        if not 1 <= q <= 100:
            raise ValueError(f"quality {quality} is outside 1..100")
        n = len(offsets)
        offsets = np.ascontiguousarray(offsets, np.int64)
        hw = np.ascontiguousarray(hw, np.int32)
        if n == 0 or (hw < 1).any() or (hw > JPEG_MAX_DIMENSION).any():
            bad = [f"{h}x{w}" for h, w in hw.tolist() if not (1 <= h <= JPEG_MAX_DIMENSION and 1 <= w <= JPEG_MAX_DIMENSION)]
            raise ValueError(f"every image must have 1..{JPEG_MAX_DIMENSION} rows and columns (libjpeg's limit), got {', '.join(bad)}")
        nbytes = ctypes.c_size_t()
        check(lib.k2y_jpeg_encode_plan(n, hw.ctypes.data_as(_INT), offsets.ctypes.data_as(_LL), q, None, 0, ctypes.byref(nbytes)))
        self.ready.synchronize()        # the previous blob copy out of the pinned buffer has finished
        if self._blob_host is None or self._blob_host.numel() < nbytes.value:
            self._blob_host = torch.empty((max(nbytes.value, 2 * (self._blob_host.numel() if self._blob_host is not None else 0)),),
                                          dtype=torch.uint8).pin_memory()
        blob = self._blob_host.numpy()
        check(lib.k2y_jpeg_encode_plan(n, hw.ctypes.data_as(_INT), offsets.ctypes.data_as(_LL), q, blob.ctypes.data, blob.size,
                                       ctypes.byref(nbytes)))
        ws, cap = ctypes.c_size_t(), ctypes.c_size_t()
        check(lib.k2y_jpeg_encode_workspace_bytes(blob.ctypes.data, ctypes.byref(ws), ctypes.byref(cap)))
        with torch.cuda.device(self.device), torch.cuda.stream(stream):
            dev = dict(dtype=torch.uint8, device=self.device)
            self._blob_dev = self._grow(self._blob_dev, nbytes.value, **dev)
            self._ws = self._grow(self._ws, ws.value, **dev)
            self.out = self._grow(self.out, cap.value, **dev)
            self._len_dev = self._grow(self._len_dev, n, dtype=torch.int64, device=self.device)
            if self.lengths_host is None or self.lengths_host.numel() < n:
                self.lengths_host = torch.empty((max(n, 32),), dtype=torch.int64).pin_memory()
            self._blob_dev[:nbytes.value].copy_(self._blob_host[:nbytes.value], non_blocking=True)
            check(lib.k2y_jpeg_encode(blob.ctypes.data, self._blob_dev.data_ptr(), ctypes.c_void_p(base_ptr), self.out.data_ptr(),
                                      self._len_dev.data_ptr(), self._ws.data_ptr(), self._ws.numel(), ctypes.c_void_p(stream.cuda_stream)))
            self.lengths_host[:n].copy_(self._len_dev[:n], non_blocking=True)
            self.ready.record(stream)
        self.n = n

    def fetch(self) -> List[bytes]:
        """The files of the last ``enqueue``, after waiting for it."""
        self.ready.synchronize()
        lengths = self.lengths_host[:self.n].numpy().astype(np.int64)
        total = int(lengths.sum())
        with torch.cuda.device(self.device):
            data = self.out[:total].cpu().numpy().tobytes()
        ends = np.cumsum(lengths)
        return [data[e - l:e] for l, e in zip(lengths.tolist(), ends.tolist())]


class JpegArgumentError(K2YError, ValueError):
    """A size or quality no JPEG file can have: a ``ValueError``, and the ``K2YError`` the library's refusal raises."""


def jpeg_header(h: int, w: int, quality: int = 75) -> bytes:
    """The marker segments (SOI .. SOS) ``encode_jpeg_batch`` writes in front of an h x w image's entropy-coded data; built on
    the host.  Raises ``JpegArgumentError`` for a size PIL cannot write (outside 1..``JPEG_MAX_DIMENSION`` rows or columns) or
    a quality outside 1..100."""
    if not (1 <= int(h) <= JPEG_MAX_DIMENSION and 1 <= int(w) <= JPEG_MAX_DIMENSION):
        raise JpegArgumentError(f"{h}x{w}: JPEG files have 1..{JPEG_MAX_DIMENSION} rows and columns (libjpeg's limit)")
    if not 1 <= int(quality) <= 100:
        raise JpegArgumentError(f"quality {quality} is outside 1..100")
    n = ctypes.c_size_t()
    check(lib.k2y_jpeg_encode_header(int(h), int(w), int(quality), None, 0, ctypes.byref(n)))
    buf = (ctypes.c_ubyte * n.value)()
    check(lib.k2y_jpeg_encode_header(int(h), int(w), int(quality), buf, n.value, ctypes.byref(n)))
    return bytes(buf)


def encode_jpeg_batch(images: Sequence[torch.Tensor], quality: int = 75, stream: Optional[torch.cuda.Stream] = None) -> List[bytes]:
    """CUDA uint8 [h, w, 3] RGB images (contiguous, e.g. what ``preprocess.decode_jpeg_batch`` returns) -> their baseline JPEG
    files, byte-identical to ``PIL.Image.fromarray(x).save(f, "JPEG", quality=quality)``.  One launch per encoding stage on
    `stream` (default: the current stream), then a synchronise and one device-to-host copy of the packed files."""
    dev, base, offsets, hw = _check_views(images)
    if not 1 <= int(quality) <= 100:
        raise ValueError(f"quality {quality} is outside 1..100")
    st = stream if stream is not None else torch.cuda.current_stream(dev)
    enc = JpegEncoder(dev)
    enc.enqueue(base, offsets, hw, quality, st)
    return enc.fetch()
