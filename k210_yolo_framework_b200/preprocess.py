"""GPU pre-processing mirror of ``Helper._process_img`` (tools/utils.py:357-406, inference branch).

``letterbox_params`` builds the affine parameters exactly as the reference does (numpy, a handful of host flops);
``letterbox_device`` runs the resampling on the GPU through the C-ABI (``k2y_letterbox_u8``, csrc/preprocess.cu) and
returns the uint8 network input; the ``img / np.max(img)`` normalisation is fused into the network's uint8 front end
(``YoloEngine.predict_device_u8``).  There is no CPU fallback: without the CUDA library the call raises.

``letterbox_batch_device`` does the same for a list of host images of different sizes in one launch: ``BatchLayout`` packs
them back to back into one pinned staging buffer (``Staging``), one H2D copy moves the whole batch and
``k2y_letterbox_u8_batch`` letterboxes every image into one uint8 [n, in_h, in_w, 3] tensor.

A batch entry may also be a whole image file (``bytes``, ``bytearray`` or ``memoryview``).  Baseline JPEGs the GPU decoder
takes (``inspect_jpeg``) travel compressed: their bytes and the batch's descriptor blob (``k2y_jpeg_plan``) go into the same
pinned buffer, one H2D copy moves them, and ``k2y_jpeg_decode`` writes their RGB pixels into the packed buffer at their
``BatchLayout`` offsets, in front of the letterbox launch, with the bytes PIL gives.  Every other file is decoded on the host
inside the call, as ``Helper._read_img`` does (the slow path); so is a JPEG that does not end with its EOI marker, so that a
truncated file raises as it does with PIL.  Corrupt entropy data in a complete file sets the image's status word, which
``letterbox_batch_device`` and ``DetectionPipeline.collect`` turn into a ``K2YError``.  ``decode_jpeg_batch`` returns the decoded pixels themselves.

PNG files take the same route when the caller opts in (``BatchLayout(gpu_png=True)``, ``letterbox_batch_device(gpu_png=True)``,
``DetectionPipeline.enable_png_decode``): the PNGs ``inspect_png`` finds GPU-decodable travel compressed in the same staging
range and H2D copy as the JPEGs, and ``k2y_png_decode`` writes the pixels PIL gives at their offsets.  A damaged zlib stream
that PIL refuses sets the image's status word (``check_png_status``).  ``decode_png_batch`` returns the decoded pixels.

Progressive JPEGs take the same route when the caller opts in (``BatchLayout(gpu_progressive=True)``,
``letterbox_batch_device(gpu_progressive=True)``, ``DetectionPipeline.enable_progressive_jpeg_decode``): the files
``progressive_gpu_decodable`` accepts travel compressed behind the JPEGs' and PNGs' ranges in the same H2D copy, and
``k2y_jpeg_progressive_decode`` writes the pixels PIL gives at their offsets (``check_progressive_status`` for corrupt data).
``decode_progressive_jpeg_batch`` returns the decoded pixels.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import numpy as np
import torch

from ._lib import JpegInfo, JpegProgressiveInfo, K2YError, PngInfo, check, lib
from .helper import read_image
from .tiles import SizedTiling, mirror_views, tile_windows, view_sides


def letterbox_params(img_hw, in_hw):
    """tools/utils.py:374-381,399: scale = min(in_wh / img_wh) on both axes, translation = ((in_wh - img_wh*scale)/2).astype(int),
    and inv(AffineTransform(scale, translation).params) — the matrix ``aff.inverse`` gives to ``skimage.transform.warp``."""
    img_wh = np.array([img_hw[1], img_hw[0]])
    in_wh = np.array([in_hw[1], in_hw[0]])
    scale = in_wh / img_wh  # NOTE affine transform scale is [w, h]
    scale[:] = np.min(scale)
    translation = ((in_wh - img_wh * scale) / 2).astype(int)
    fwd = np.array([[scale[0], 0.0, float(translation[0])], [0.0, scale[1], float(translation[1])], [0.0, 0.0, 1.0]])
    return scale, translation, np.linalg.inv(fwd)


def letterbox_device(img_u8: torch.Tensor, in_hw, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """img_u8: CUDA uint8 [h, w, 3] RGB of any size -> CUDA uint8 [in_h, in_w, 3] letterboxed (zero fill)."""
    if img_u8.dim() != 3 or img_u8.shape[2] != 3 or img_u8.dtype != torch.uint8 or not img_u8.is_cuda:
        raise ValueError(f"expected CUDA uint8 [h,w,3], got {tuple(img_u8.shape)} {img_u8.dtype} {img_u8.device}")
    img_u8 = img_u8.contiguous()
    in_h, in_w = int(in_hw[0]), int(in_hw[1])
    if out is None:
        out = torch.empty((in_h, in_w, 3), dtype=torch.uint8, device=img_u8.device)
    elif tuple(out.shape) != (in_h, in_w, 3) or out.dtype != torch.uint8 or out.device != img_u8.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous CUDA uint8 [in_h,in_w,3] tensor on the image's device")
    _, _, inv = letterbox_params(img_u8.shape[:2], (in_h, in_w))
    m = (ctypes.c_double * 6)(*[float(v) for v in inv[:2].reshape(-1)])
    minmax = torch.empty((2,), dtype=torch.int32, device=img_u8.device)
    with torch.cuda.device(img_u8.device):
        st = torch.cuda.current_stream()
        check(lib.k2y_letterbox_u8(img_u8.data_ptr(), int(img_u8.shape[0]), int(img_u8.shape[1]), m, out.data_ptr(), in_h, in_w,
                                   minmax.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
    return out


ALIGN = 16   # byte alignment of each packed image (pass 1 of the batch kernel then reads 16 bytes at a time)


ENCODED = (bytes, bytearray, memoryview)


def _file_bytes(data) -> np.ndarray:
    """A whole image file as a read-only uint8 array over the caller's buffer (no copy)."""
    return np.frombuffer(data, dtype=np.uint8)


def _jpeg_info(buf: np.ndarray) -> Optional[JpegInfo]:
    """The header of a JPEG file, or None when `buf` is not one the parser accepts (other formats, malformed headers)."""
    if buf.size < 4 or buf[0] != 0xFF or buf[1] != 0xD8:
        return None
    info = JpegInfo()
    if lib.k2y_jpeg_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)) != 0:
        return None
    return info


def inspect_jpeg(data):
    """Header of a JPEG file held in memory (``bytes``, ``bytearray`` or ``memoryview``), read on the host:
    ``(h, w, gpu_decodable, reason)``; `reason` says why a valid file is not for the GPU decoder ("" when it is).
    Raises ``K2YError`` for a file that is not a JPEG or whose headers are malformed (the message names the marker)."""
    if not isinstance(data, ENCODED):
        raise ValueError(f"expected the bytes of a file, got {type(data).__name__}")
    buf = _file_bytes(data)
    info = JpegInfo()
    check(lib.k2y_jpeg_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)))
    return int(info.height), int(info.width), bool(info.gpu_decodable), info.reason.decode()


def _gpu_route(buf: np.ndarray) -> Optional[JpegInfo]:
    """The header of `buf` when the batch routes send it to the GPU decoder, else None.  A file must be GPU-decodable and end
    with its EOI marker: a truncated file (or one with data appended after EOI) goes to the host decoder, which reports the
    truncation as PIL does instead of decoding pixels the missing data would have set."""
    info = _jpeg_info(buf)
    if info is None or not info.gpu_decodable or buf[-2] != 0xFF or buf[-1] != 0xD9:
        return None
    return info


def gpu_decodable(data) -> bool:
    """True when `data` (the bytes of a file) goes to the GPU decoder in ``submit_images``: a JPEG the decoder takes, ending
    with its EOI marker.  False for anything else, malformed or truncated files included."""
    return _gpu_route(_file_bytes(data)) is not None


def _progressive_info(buf: np.ndarray) -> Optional[JpegProgressiveInfo]:
    """What the progressive walk says of a JPEG file, or None when `buf` is not one it accepts (other formats, malformed
    headers or scans)."""
    if buf.size < 4 or buf[0] != 0xFF or buf[1] != 0xD8:
        return None
    info = JpegProgressiveInfo()
    if lib.k2y_jpeg_progressive_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)) != 0:
        return None
    return info


def inspect_jpeg_progressive(data):
    """``inspect_jpeg`` for the progressive decoder: ``(h, w, gpu_decodable, reason)``, where `reason` says why a valid file is
    not for the GPU progressive decoder ("sequential (SOF 0xC0)" for a baseline file, a script libjpeg-turbo warns about or
    would block-smooth, ...).  Walks every marker to EOI.  Raises ``K2YError`` for a file that is not a JPEG or whose headers
    or scan parameters are malformed (the message names the marker or the scan)."""
    if not isinstance(data, ENCODED):
        raise ValueError(f"expected the bytes of a file, got {type(data).__name__}")
    buf = _file_bytes(data)
    info = JpegProgressiveInfo()
    check(lib.k2y_jpeg_progressive_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)))
    return int(info.height), int(info.width), bool(info.gpu_decodable), info.reason.decode()


def _progressive_route(buf: np.ndarray) -> Optional[JpegProgressiveInfo]:
    """The header of `buf` when the batch routes send it to the GPU progressive decoder (with progressive decoding enabled):
    GPU-decodable and ending with its EOI marker, as for baseline files (``_gpu_route``)."""
    info = _progressive_info(buf)
    if info is None or not info.gpu_decodable or buf[-2] != 0xFF or buf[-1] != 0xD9:
        return None
    return info


def progressive_gpu_decodable(data) -> bool:
    """True when `data` (the bytes of a file) goes to the GPU progressive decoder in ``submit_images`` with progressive
    decoding enabled."""
    return _progressive_route(_file_bytes(data)) is not None


def _png_info(buf: np.ndarray) -> Optional[PngInfo]:
    """The header of a PNG file, or None when `buf` is not one the parser accepts (other formats, no sound IHDR)."""
    if buf.size < 8 or bytes(buf[:8]) != b"\x89PNG\r\n\x1a\n":
        return None
    info = PngInfo()
    if lib.k2y_png_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)) != 0:
        return None
    return info


def _pil_pixel_limit() -> Optional[int]:
    from PIL import Image
    return Image.MAX_IMAGE_PIXELS


def inspect_png(data):
    """Header of a PNG file held in memory (``bytes``, ``bytearray`` or ``memoryview``), read on the host:
    ``(h, w, gpu_decodable, reason)``; `reason` says why a valid file is not for the GPU decoder ("" when it is).  A file over
    PIL's decompression-bomb limit (``Image.MAX_IMAGE_PIXELS``) is left to PIL, which warns or raises.  Raises ``K2YError``
    for a file that is not a PNG or has no sound IHDR chunk."""
    if not isinstance(data, ENCODED):
        raise ValueError(f"expected the bytes of a file, got {type(data).__name__}")
    buf = _file_bytes(data)
    info = PngInfo()
    check(lib.k2y_png_inspect(buf.ctypes.data, buf.size, ctypes.byref(info)))
    h, w, ok, why = int(info.height), int(info.width), bool(info.gpu_decodable), info.reason.decode()
    limit = _pil_pixel_limit()
    if ok and limit is not None and h * w > limit:
        ok, why = False, f"over PIL's decompression-bomb limit of {limit} pixels"
    return h, w, ok, why


def _png_route(buf: np.ndarray) -> Optional[PngInfo]:
    """The header of `buf` when the batch routes send it to the GPU PNG decoder (with PNG decoding enabled), else None."""
    info = _png_info(buf)
    if info is None or not info.gpu_decodable:
        return None
    limit = _pil_pixel_limit()
    if limit is not None and int(info.height) * int(info.width) > limit:
        return None
    return info


def png_gpu_decodable(data) -> bool:
    """True when `data` (the bytes of a file) goes to the GPU PNG decoder in ``submit_images`` with PNG decoding enabled."""
    return _png_route(_file_bytes(data)) is not None


def _check_images(images) -> None:
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("expected a non-empty list of host uint8 [h, w, 3] arrays or image files")
    for i, im in enumerate(images):
        if isinstance(im, ENCODED):
            if not memoryview(im).c_contiguous:
                raise ValueError(f"image {i}: the memoryview of a file must be contiguous")
            if memoryview(im).nbytes == 0:
                raise ValueError(f"image {i}: empty file")
            continue
        if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
            desc = f"{im.dtype} {im.shape}" if isinstance(im, np.ndarray) else type(im).__name__
            raise ValueError(f"image {i}: expected a host numpy uint8 [h, w, 3] array or the bytes of an image file, got {desc}")


def _host_decode(buf: np.ndarray, i: int) -> np.ndarray:
    import io
    try:
        return read_image(io.BytesIO(buf.tobytes()))
    except Exception as e:  # PIL raises several types for unreadable files
        raise ValueError(f"image {i}: cannot decode the file: {e}") from e


class BatchLayout:
    """Where each image of a ragged batch lies in the packed buffer, and its letterbox descriptor.

    ``offsets`` int64 [n] (multiples of ``ALIGN``), ``hw`` int32 [n, 2] (h, w), ``matrices`` float64 [n, 6] (the first two
    rows of ``letterbox_params``' inverse matrix), ``nbytes`` the packed size.

    Entries that are image files are resolved here: ``jpeg`` lists (index, file bytes) of the JPEGs the GPU decodes
    (``gpu_decodable``), whose size comes from their header; every other file is decoded on the host now, and ``arrays[i]``
    holds the host pixels of entry i (None for a GPU JPEG).  ``jpeg_plan`` is where the JPEGs' bytes and their descriptor blob
    go in the staging buffer, behind the packed pixels (``_jpeg_layout``).  With `gpu_png`, ``png`` lists (index, file bytes) of
    the PNGs the GPU decodes (``png_gpu_decodable``) in the same way, and ``png_plan`` places them and their blob behind the
    JPEGs' range, so that one H2D copy moves both (``staged_end`` is the end of everything the staging buffer holds).  With
    `gpu_progressive`, ``progressive`` and ``progressive_plan`` do the same for the progressive JPEGs the GPU decodes
    (``progressive_gpu_decodable``), behind the PNGs' range.

    With `tiling` = (rows, cols, overlap) every image is letterboxed as V = 1 + rows * cols views (``tiles.tile_windows``:
    the whole image, then its tiles): ``views`` = V, ``windows`` int32 [n * V, 4] (y0, x0, th, tw) and ``view_matrices``
    float64 [n * V, 6] (each window's own ``letterbox_params`` matrix), image-major.  Everything above stays per image: staging,
    the JPEG decode and the renderer see the originals.  `tiling` may also be a ``tiles.SizedTiling``, whose grid is planned
    per image (``tiles.plan_windows``); ``views`` is then None.  Either way ``view_counts`` int32 [n] holds each image's number
    of views, ``view_offsets`` int32 [n + 1] their running sum (image b's views are ``windows[view_offsets[b]:view_offsets[b+1]]``)
    and ``view_sides`` int32 [N] each window's interior sides (``tiles.view_sides``).

    With `flip` (with or without a tiling) each image's W windows (the whole image alone without a tiling) are followed by
    the same W windows mirrored (``tiles.mirror_views``): ``view_mirror`` int32 [N] flags them, and their ``view_sides`` are
    their windows' (the merge swaps left and right for a mirrored view).  Without `flip` ``view_mirror`` is None.

    With `merge_table` (and a tiling or flip) ``view_offsets``, ``view_sides`` and, with `flip`, ``view_mirror`` also go into
    the staging buffer, behind everything else, at ``merge_table_at``, so that the batch's H2D copy takes them to the device
    for ``k2y_merge_views_ex`` / ``k2y_merge_views_mirror``."""

    def __init__(self, images: Sequence, in_hw, tiling=None, gpu_png: bool = False, gpu_progressive: bool = False,
                 merge_table: bool = False, flip: bool = False):
        _check_images(images)
        n = len(images)
        self.in_hw = (int(in_hw[0]), int(in_hw[1]))
        self.arrays: List[Optional[np.ndarray]] = []
        self.jpeg = []
        self.png = []
        self.progressive = []
        shapes = []
        for i, im in enumerate(images):
            if isinstance(im, ENCODED):
                buf = _file_bytes(im)
                info = _gpu_route(buf)
                to = self.jpeg
                if info is None and gpu_png:
                    info, to = _png_route(buf), self.png
                if info is None and gpu_progressive:
                    info, to = _progressive_route(buf), self.progressive
                if info is not None:
                    to.append((i, buf))
                    self.arrays.append(None)
                    shapes.append((info.height, info.width))
                    continue
                im = _host_decode(buf, i)
            self.arrays.append(im)
            shapes.append(im.shape[:2])
        self.hw = np.array(shapes, dtype=np.int32).reshape(n, 2)
        sizes = self.hw[:, 0].astype(np.int64) * self.hw[:, 1] * 3
        padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
        self.offsets = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
        self.nbytes = int(padded.sum())
        self.matrices = np.array([letterbox_params((int(h[0]), int(h[1])), self.in_hw)[2][:2].reshape(-1) for h in self.hw], dtype=np.float64)
        self.views, self.windows, self.view_matrices = 1, None, None
        self.view_counts, self.view_offsets, self.view_sides, self.view_mirror = None, None, None, None
        if tiling is not None or flip:
            if tiling is None:
                what, plan = "flip", lambda h, w: np.array([(0, 0, h, w)], np.int32)      # noqa: E731
            elif isinstance(tiling, (tuple, list)):
                rows, cols, overlap = tiling
                what = f"tiling {rows}x{cols}"
                plan = lambda h, w: tile_windows(h, w, rows, cols, overlap)     # noqa: E731
            else:
                what, plan = f"tiling by {tiling.tile_hw[0]}x{tiling.tile_hw[1]} tiles", tiling.windows
            try:
                per_image = [plan(int(h), int(w)) for h, w in self.hw]
            except ValueError as e:
                raise ValueError(f"{what}: {e}") from e
            if flip:
                per_image, mirror = zip(*[mirror_views(w) for w in per_image])
                self.view_mirror = np.concatenate(mirror)
            self.windows = np.concatenate(per_image)
            self.view_counts = np.array([len(w) for w in per_image], np.int32)
            self.view_offsets = np.concatenate([[0], np.cumsum(self.view_counts)]).astype(np.int32)
            self.view_sides = np.concatenate([view_sides(w, int(h), int(wd)) for w, (h, wd) in zip(per_image, self.hw)])
            self.views = None if isinstance(tiling, SizedTiling) else len(self.windows) // n
            self.view_matrices = np.array([letterbox_params((int(t[2]), int(t[3])), self.in_hw)[2][:2].reshape(-1) for t in self.windows],
                                          dtype=np.float64)
        self.jpeg_plan = None
        self.png_plan = None
        self.progressive_plan = None
        self.staged_end = self.nbytes
        if self.jpeg:
            self.jpeg_dst = self.offsets[[i for i, _ in self.jpeg]].astype(np.int64)
            self.jpeg_plan = _jpeg_layout([f for _, f in self.jpeg], self.jpeg_dst, (self.nbytes + ALIGN - 1) // ALIGN * ALIGN)
            self.staged_end = self.jpeg_plan[3]
        if self.png:
            self.png_dst = self.offsets[[i for i, _ in self.png]].astype(np.int64)
            self.png_plan = _jpeg_layout([f for _, f in self.png], self.png_dst, (self.staged_end + ALIGN - 1) // ALIGN * ALIGN,
                                         _png_plan)
            self.staged_end = self.png_plan[3]
        if self.progressive:
            self.progressive_dst = self.offsets[[i for i, _ in self.progressive]].astype(np.int64)
            self.progressive_plan = _jpeg_layout([f for _, f in self.progressive], self.progressive_dst,
                                                 (self.staged_end + ALIGN - 1) // ALIGN * ALIGN, _progressive_plan)
            self.staged_end = self.progressive_plan[3]
        self.merge_table_at = None
        if merge_table and self.windows is not None:
            self.merge_table = np.concatenate([self.view_offsets, self.view_sides] +
                                              ([] if self.view_mirror is None else [self.view_mirror])).astype(np.int32)
            self.merge_table_at = (self.staged_end + ALIGN - 1) // ALIGN * ALIGN
            self.staged_end = self.merge_table_at + self.merge_table.nbytes

    @property
    def n_views(self) -> int:
        """Network inputs of the batch: one per image, or every image's views with a tiling."""
        return len(self.hw) if self.windows is None else len(self.windows)

    def __len__(self) -> int:
        return len(self.hw)

    def pack(self, images: Sequence, host: np.ndarray) -> None:
        """Copies the host pixels of `images` (the entries this layout was made of) into the uint8 buffer `host` (at least
        ``nbytes`` long) at their offsets.  The GPU JPEGs' ranges are left as they are: the decoder fills them on the device."""
        assert len(images) == len(self.arrays)
        for im, off, (h, w) in zip(self.arrays, self.offsets, self.hw):
            if im is not None:
                np.copyto(host[off:off + h * w * 3].reshape(h, w, 3), im)

    def host_ranges(self):
        """[begin, end) ranges of the packed buffer that hold the host-side images, one per run of consecutive ones (the GPU
        JPEGs' ranges between them are filled on the device and need no copy)."""
        out = []
        for i, a in enumerate(self.arrays):
            if a is None:
                continue
            b, e = int(self.offsets[i]), int(self.offsets[i] + self.hw[i, 0] * self.hw[i, 1] * 3)
            if out and self.arrays[i - 1] is not None:
                out[-1] = (out[-1][0], e)
            else:
                out.append((b, e))
        return out


class Staging:
    """A pinned host buffer and a device buffer for packed batches, plus the kernel's min/max scratch, reused across calls.
    They grow (geometrically) only when a batch does not fit; the caller makes sure the previous H2D copy out of the host
    buffer has finished first.  The device buffers are allocated on `stream`, the stream that reads them."""

    def __init__(self, device: torch.device, stream: torch.cuda.Stream):
        self.device, self.stream = device, stream
        self.host: Optional[torch.Tensor] = None
        self.dev: Optional[torch.Tensor] = None
        self.minmax: Optional[torch.Tensor] = None
        self.workspace: Optional[torch.Tensor] = None   # k2y_jpeg_decode's
        self.status: Optional[torch.Tensor] = None      # int32 [n, 4] per decoded JPEG (k2y_jpeg_decode)
        self.png_workspace: Optional[torch.Tensor] = None   # k2y_png_decode's
        self.png_status: Optional[torch.Tensor] = None      # int32 [n, 4] per decoded PNG (k2y_png_decode)
        self.progressive_workspace: Optional[torch.Tensor] = None   # k2y_jpeg_progressive_decode's
        self.progressive_status: Optional[torch.Tensor] = None      # int32 [n, 4] per decoded progressive JPEG

    def reserve_progressive(self, workspace_bytes: int, n: int) -> None:
        with torch.cuda.stream(self.stream):
            ws, st = self.progressive_workspace, self.progressive_status
            if ws is None or ws.numel() < workspace_bytes:
                cap = max(workspace_bytes, 2 * ws.numel() if ws is not None else 0)
                self.progressive_workspace = torch.empty((cap,), dtype=torch.uint8, device=self.device)
            if st is None or st.shape[0] < n:
                self.progressive_status = torch.empty((max(n, 2 * st.shape[0] if st is not None else 0), 4), dtype=torch.int32,
                                                      device=self.device)

    def reserve_jpeg(self, workspace_bytes: int, n: int) -> None:
        with torch.cuda.stream(self.stream):
            if self.workspace is None or self.workspace.numel() < workspace_bytes:
                cap = max(workspace_bytes, 2 * self.workspace.numel() if self.workspace is not None else 0)
                self.workspace = torch.empty((cap,), dtype=torch.uint8, device=self.device)
            if self.status is None or self.status.shape[0] < n:
                self.status = torch.empty((max(n, 2 * self.status.shape[0] if self.status is not None else 0), 4), dtype=torch.int32,
                                          device=self.device)

    def reserve_png(self, workspace_bytes: int, n: int) -> None:
        with torch.cuda.stream(self.stream):
            if self.png_workspace is None or self.png_workspace.numel() < workspace_bytes:
                cap = max(workspace_bytes, 2 * self.png_workspace.numel() if self.png_workspace is not None else 0)
                self.png_workspace = torch.empty((cap,), dtype=torch.uint8, device=self.device)
            if self.png_status is None or self.png_status.shape[0] < n:
                self.png_status = torch.empty((max(n, 2 * self.png_status.shape[0] if self.png_status is not None else 0), 4),
                                              dtype=torch.int32, device=self.device)

    def reserve(self, nbytes: int, n: int) -> None:
        if self.host is None or self.host.numel() < nbytes:
            cap = max(nbytes, 2 * self.host.numel() if self.host is not None else 0)
            self.host = torch.empty((cap,), dtype=torch.uint8, pin_memory=True)
            with torch.cuda.stream(self.stream):
                self.dev = torch.empty((cap,), dtype=torch.uint8, device=self.device)
        if self.minmax is None or self.minmax.shape[0] < n:
            with torch.cuda.stream(self.stream):
                self.minmax = torch.empty((max(n, 2 * self.minmax.shape[0] if self.minmax is not None else 0), 2), dtype=torch.int32,
                                          device=self.device)


def _check_out(t: Optional[torch.Tensor], n: int, shape, dtype, name: str, device) -> None:
    if t is None:
        return
    if (not t.is_cuda or t.dtype != dtype or not t.is_contiguous() or t.dim() != 1 + len(shape) or tuple(t.shape[1:]) != tuple(shape)
            or (device is not None and t.device != device)):
        raise ValueError(f"{name} must be a contiguous CUDA {dtype} [N, {', '.join(map(str, shape))}] tensor")
    if t.shape[0] < n:
        raise ValueError(f"{n} images do not fit {name}, which holds {t.shape[0]}")


def _jpeg_plan(files: Sequence[np.ndarray], src_offsets: np.ndarray, dst_offsets: np.ndarray, blob: Optional[np.ndarray]) -> int:
    """k2y_jpeg_plan: the blob's size (blob None), or the blob written into `blob` (16-byte aligned)."""
    n = len(files)
    ptrs = (ctypes.c_void_p * n)(*[f.ctypes.data for f in files])
    sizes = (ctypes.c_size_t * n)(*[f.size for f in files])
    nbytes = ctypes.c_size_t()
    ll = ctypes.POINTER(ctypes.c_longlong)
    check(lib.k2y_jpeg_plan(ptrs, sizes, n, src_offsets.ctypes.data_as(ll), dst_offsets.ctypes.data_as(ll),
                            blob.ctypes.data if blob is not None else None, blob.size if blob is not None else 0, ctypes.byref(nbytes)))
    return nbytes.value


def _png_plan(files: Sequence[np.ndarray], src_offsets: np.ndarray, dst_offsets: np.ndarray, blob: Optional[np.ndarray]) -> int:
    """k2y_png_plan: the blob's size (blob None), or the blob written into `blob` (16-byte aligned)."""
    n = len(files)
    ptrs = (ctypes.c_void_p * n)(*[f.ctypes.data for f in files])
    sizes = (ctypes.c_size_t * n)(*[f.size for f in files])
    nbytes = ctypes.c_size_t()
    ll = ctypes.POINTER(ctypes.c_longlong)
    check(lib.k2y_png_plan(ptrs, sizes, n, src_offsets.ctypes.data_as(ll), dst_offsets.ctypes.data_as(ll),
                           blob.ctypes.data if blob is not None else None, blob.size if blob is not None else 0, ctypes.byref(nbytes)))
    return nbytes.value


def _progressive_plan(files: Sequence[np.ndarray], src_offsets: np.ndarray, dst_offsets: np.ndarray, blob: Optional[np.ndarray]) -> int:
    """k2y_jpeg_progressive_plan: the blob's size (blob None), or the blob written into `blob` (16-byte aligned)."""
    n = len(files)
    ptrs = (ctypes.c_void_p * n)(*[f.ctypes.data for f in files])
    sizes = (ctypes.c_size_t * n)(*[f.size for f in files])
    nbytes = ctypes.c_size_t()
    ll = ctypes.POINTER(ctypes.c_longlong)
    check(lib.k2y_jpeg_progressive_plan(ptrs, sizes, n, src_offsets.ctypes.data_as(ll), dst_offsets.ctypes.data_as(ll),
                                        blob.ctypes.data if blob is not None else None, blob.size if blob is not None else 0,
                                        ctypes.byref(nbytes)))
    return nbytes.value


_DECODERS = {"jpeg": (_jpeg_plan, "k2y_jpeg_workspace_bytes", "k2y_jpeg_decode", "reserve_jpeg", "workspace", "status"),
             "png": (_png_plan, "k2y_png_workspace_bytes", "k2y_png_decode", "reserve_png", "png_workspace", "png_status"),
             "progressive": (_progressive_plan, "k2y_jpeg_progressive_workspace_bytes", "k2y_jpeg_progressive_decode",
                             "reserve_progressive", "progressive_workspace", "progressive_status")}


def _fill(kind: str, files: Sequence[np.ndarray], dst_offsets: np.ndarray, staging: Staging, plan):
    """Writes `files` and their blob into ``staging.host`` where `plan` places them and reserves the decode's workspace and
    status words; returns the decode call, to be enqueued once the range is on the device."""
    planner, ws_fn, decode_fn, reserve, ws_name, status_name = _DECODERS[kind]
    src_offsets, blob_at, blob_bytes, end = plan
    host = staging.host.numpy()
    for f, off in zip(files, src_offsets):
        host[off:off + f.size] = f
    blob = host[blob_at:blob_at + blob_bytes]
    planner(files, src_offsets, dst_offsets, blob)
    ws = ctypes.c_size_t()
    check(getattr(lib, ws_fn)(blob.ctypes.data, ctypes.byref(ws)))
    getattr(staging, reserve)(ws.value, len(files))
    workspace, status = getattr(staging, ws_name), getattr(staging, status_name)

    def decode(dst: torch.Tensor):
        st = staging.stream
        with torch.cuda.stream(st):
            check(getattr(lib, decode_fn)(blob.ctypes.data, staging.dev.data_ptr() + blob_at, staging.dev.data_ptr(), dst.data_ptr(),
                                          workspace.data_ptr(), workspace.numel(), status.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
    return decode


def _stage(kind: str, files: Sequence[np.ndarray], dst_offsets: np.ndarray, staging: Staging, plan, dst: torch.Tensor) -> None:
    decode = _fill(kind, files, dst_offsets, staging, plan)
    b, e = int(plan[0][0]), plan[3]
    with torch.cuda.stream(staging.stream):
        staging.dev[b:e].copy_(staging.host[b:e], non_blocking=True)
    decode(dst)


def stage_jpegs(files: Sequence[np.ndarray], dst_offsets: np.ndarray, staging: Staging, plan, dst: torch.Tensor) -> None:
    """Puts the JPEG `files` and their descriptor blob into ``staging.host`` where `plan` (``_jpeg_layout``) places them
    (``staging.reserve`` of the whole batch first), copies that range to ``staging.dev`` in one H2D copy and decodes the files
    into `dst` (a device uint8 buffer) at `dst_offsets`, on ``staging.stream``.  Per-image status words land in
    ``staging.status``."""
    _stage("jpeg", files, dst_offsets, staging, plan, dst)


def stage_progressive_jpegs(files: Sequence[np.ndarray], dst_offsets: np.ndarray, staging: Staging, plan, dst: torch.Tensor) -> None:
    """``stage_jpegs`` for GPU-decodable progressive JPEG files (`plan` from ``_jpeg_layout(..., _progressive_plan)``); status
    words land in ``staging.progressive_status``."""
    _stage("progressive", files, dst_offsets, staging, plan, dst)


def stage_pngs(files: Sequence[np.ndarray], dst_offsets: np.ndarray, staging: Staging, plan, dst: torch.Tensor) -> None:
    """``stage_jpegs`` for GPU-decodable PNG files (`plan` from ``_jpeg_layout(..., _png_plan)``); status words land in
    ``staging.png_status``."""
    _stage("png", files, dst_offsets, staging, plan, dst)


def _jpeg_layout(files: Sequence[np.ndarray], dst_offsets: np.ndarray, base: int, planner=_jpeg_plan):
    """Offsets of the files and of the blob in the staging buffer from `base` on, the blob's size and the end of the range.
    The blob's size query parses every header: a file the plan refuses raises ``ValueError`` here.  `planner`: ``_jpeg_plan``,
    ``_png_plan`` or ``_progressive_plan``."""
    sizes = np.array([f.size for f in files], np.int64)
    padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
    src_offsets = (base + np.concatenate([[0], np.cumsum(padded)[:-1]])).astype(np.int64)
    blob_at = int(base + padded.sum())
    try:
        blob_bytes = planner(files, src_offsets, dst_offsets, None)
    except K2YError as e:
        raise ValueError(str(e)) from e
    return src_offsets, blob_at, blob_bytes, blob_at + blob_bytes


def letterbox_packed(layout: BatchLayout, images: Sequence, staging: Staging, out: torch.Tensor,
                     image_hw_out: Optional[torch.Tensor], view_yx_out: Optional[torch.Tensor] = None) -> None:
    """Packs `images` into ``staging.host``, copies them to the device and letterboxes them into ``out[:n]`` (and their sizes
    into ``image_hw_out[:n]``), all on ``staging.stream``.  GPU-decodable JPEGs travel compressed behind the packed pixels and
    are decoded into their place first (``stage_jpegs``), and so are the layout's GPU PNGs, whose range the same H2D copy moves
    (``stage_pngs``).  The host buffer is reused by the next call: wait for this copy
    before packing into it again.  A layout with tiling letterboxes its N = ``layout.n_views`` views instead
    (``k2y_letterbox_u8_views_mirror``, the mirrored ones flipped left to right), image-major: ``out[:N]``, each view's (th, tw) into ``image_hw_out[:N]`` and its (y0, x0) into
    ``view_yx_out[:N]`` (float32 [N, 2]); a layout's merge table goes to ``staging.dev`` at ``layout.merge_table_at`` in the
    same H2D copy as the rest."""
    n = len(layout)
    staging.reserve(layout.staged_end, layout.n_views)
    layout.pack(images, staging.host.numpy())
    ranges = layout.host_ranges()
    table = layout.merge_table_at is not None
    if table:       # the merge table rides along with the last H2D copy: the decoders' range, else the last host range
        at = layout.merge_table_at
        staging.host.numpy()[at:at + layout.merge_table.nbytes] = layout.merge_table.view(np.uint8)
        if not (layout.jpeg or layout.png or layout.progressive):
            ranges[-1] = (ranges[-1][0], layout.staged_end)
    in_h, in_w = layout.in_hw
    st = staging.stream
    with torch.cuda.stream(st):
        for b, e in ranges:
            staging.dev[b:e].copy_(staging.host[b:e], non_blocking=True)
        if layout.png or layout.progressive or (layout.jpeg and table):   # every decoder's files and blobs in one H2D copy
            decodes = [_fill(k, [f for _, f in files], dst, staging, plan) for k, files, dst, plan in
                       (("jpeg", layout.jpeg, getattr(layout, "jpeg_dst", None), layout.jpeg_plan),
                        ("png", layout.png, getattr(layout, "png_dst", None), layout.png_plan),
                        ("progressive", layout.progressive, getattr(layout, "progressive_dst", None), layout.progressive_plan))
                       if files]
            b = int((layout.jpeg_plan or layout.png_plan or layout.progressive_plan)[0][0])
            staging.dev[b:layout.staged_end].copy_(staging.host[b:layout.staged_end], non_blocking=True)
            for decode in decodes:
                decode(staging.dev)
        elif layout.jpeg:
            stage_jpegs([f for _, f in layout.jpeg], layout.jpeg_dst, staging, layout.jpeg_plan, staging.dev)
        offs = layout.offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong))
        if layout.windows is not None:
            offsets = np.repeat(layout.offsets, layout.view_counts)
            hw = np.ascontiguousarray(np.repeat(layout.hw, layout.view_counts, axis=0))
            mirror = None if layout.view_mirror is None else layout.view_mirror.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
            check(lib.k2y_letterbox_u8_views_mirror(staging.dev.data_ptr(), layout.n_views,
                                                    offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                                    hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                                    layout.windows.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), mirror,
                                                    layout.view_matrices.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), out.data_ptr(),
                                                    in_h, in_w, image_hw_out.data_ptr() if image_hw_out is not None else None,
                                                    view_yx_out.data_ptr() if view_yx_out is not None else None,
                                                    staging.minmax.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
            return
        hw = layout.hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
        mats = layout.matrices.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        check(lib.k2y_letterbox_u8_batch(staging.dev.data_ptr(), n, offs, hw, mats, out.data_ptr(), in_h, in_w,
                                         image_hw_out.data_ptr() if image_hw_out is not None else None, staging.minmax.data_ptr(),
                                         ctypes.c_void_p(st.cuda_stream)))


def letterbox_batch_device(images: List, in_hw, out: Optional[torch.Tensor] = None,
                           image_hw_out: Optional[torch.Tensor] = None, stream: Optional[torch.cuda.Stream] = None,
                           gpu_png: bool = False, gpu_progressive: bool = False) -> torch.Tensor:
    """images: host numpy uint8 [h, w, 3] RGB arrays of any sizes, or image files (``bytes``, ``bytearray``, ``memoryview``:
    see ``BatchLayout``) -> CUDA uint8 [n, in_h, in_w, 3] letterboxed (zero fill), the
    same bytes ``letterbox_device`` gives each image.  One pinned staging buffer, one H2D copy, one batched letterbox launch on
    `stream` (default: the current stream), asynchronous.  `out` ([N >= n, in_h, in_w, 3] uint8, e.g. a network's bound input)
    receives the images in its first n rows; `image_hw_out` ([N >= n, 2] float32), if given, receives each image's (h, w).
    When the batch holds JPEGs decoded on the GPU, the call synchronises `stream` to read their status words and raises
    ``K2YError`` if one of them was corrupt (``check_jpeg_status``).  With `gpu_png` the PNGs the GPU takes are decoded there
    too (``BatchLayout``), and a damaged zlib stream PIL refuses raises the same way (``check_png_status``); so do the
    progressive JPEGs with `gpu_progressive` (``check_progressive_status``)."""
    in_h, in_w = int(in_hw[0]), int(in_hw[1])
    layout = BatchLayout(images, (in_h, in_w), gpu_png=gpu_png, gpu_progressive=gpu_progressive)
    n = len(layout)
    device = out.device if out is not None else torch.device("cuda", torch.cuda.current_device())
    _check_out(out, n, (in_h, in_w, 3), torch.uint8, "out", None)
    _check_out(image_hw_out, n, (2,), torch.float32, "image_hw_out", device)
    st = stream if stream is not None else torch.cuda.current_stream(device)
    if out is None:
        with torch.cuda.stream(st):
            out = torch.empty((n, in_h, in_w, 3), dtype=torch.uint8, device=device)
    staging = Staging(device, st)
    with torch.cuda.device(device):
        letterbox_packed(layout, images, staging, out, image_hw_out)
        if layout.jpeg or layout.png or layout.progressive:
            with torch.cuda.stream(st):
                jst = staging.status[:len(layout.jpeg)].cpu().numpy() if layout.jpeg else None
                pst = staging.png_status[:len(layout.png)].cpu().numpy() if layout.png else None
                gst = staging.progressive_status[:len(layout.progressive)].cpu().numpy() if layout.progressive else None
            if layout.jpeg:
                check_jpeg_status(jst, [i for i, _ in layout.jpeg])
            if layout.png:
                check_png_status(pst, [i for i, _ in layout.png])
            if layout.progressive:
                check_progressive_status(gst, [i for i, _ in layout.progressive])
    return out


def decode_jpeg_batch(files: Sequence, stream: Optional[torch.cuda.Stream] = None, with_status: bool = False):
    """GPU-decodable JPEG files (``bytes``, ``bytearray``, ``memoryview``) -> list of CUDA uint8 [h, w, 3] RGB views of one
    packed device buffer, byte for byte what ``Helper._read_img`` (PIL) gives.  One pinned staging buffer, one H2D copy and
    one launch per decode stage on `stream` (default: the current stream), then a synchronise to read the per-image status.
    A file the GPU decoder does not take raises ``ValueError`` before anything is enqueued; corrupt entropy data raises
    ``K2YError`` naming the images, unless `with_status`, which returns (views, status int32 [n, 4]: error bits, max / sum of
    synchronisation rounds per window, windows) instead."""
    if not isinstance(files, (list, tuple)) or len(files) == 0:
        raise ValueError("expected a non-empty list of JPEG files")
    bufs, shapes = [], []
    for i, f in enumerate(files):
        if not isinstance(f, ENCODED):
            raise ValueError(f"file {i}: expected bytes, bytearray or memoryview, got {type(f).__name__}")
        buf = _file_bytes(f)
        info = _jpeg_info(buf)
        if info is None or not info.gpu_decodable:
            why = info.reason.decode() if info is not None else "not a well-formed JPEG file"
            raise ValueError(f"file {i}: not decodable on the GPU: {why}")
        bufs.append(buf)
        shapes.append((int(info.height), int(info.width)))
    sizes = np.array([h * w * 3 for h, w in shapes], np.int64)
    padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
    offsets = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    device = torch.device("cuda", torch.cuda.current_device())
    st = stream if stream is not None else torch.cuda.current_stream(device)
    staging = Staging(device, st)
    plan = _jpeg_layout(bufs, offsets, int(padded.sum()))
    staging.reserve(plan[3], len(bufs))
    with torch.cuda.stream(st):
        stage_jpegs(bufs, offsets, staging, plan, staging.dev)
        status = staging.status[:len(bufs)].cpu().numpy()
    out = [staging.dev[o:o + h * w * 3].view(h, w, 3) for o, (h, w) in zip(offsets, shapes)]
    if with_status:
        return out, status
    check_jpeg_status(status, range(len(bufs)))
    return out


def check_jpeg_status(status: np.ndarray, images) -> None:
    """Raises ``K2YError`` naming the images whose entropy-coded data was corrupt, ended early or had its restart markers out
    of sequence.  `status`: the decode's int32 [n, 4] words of the GPU-decoded JPEGs, `images`: their positions in the
    caller's batch."""
    bad = [(int(i), int(w)) for i, w in zip(images, status[:, 0]) if w]
    if bad:
        raise K2YError("corrupt JPEG data: " + ", ".join(
            f"image {i}: " + ", ".join(v for k, v in JPEG_ERRORS.items() if w & k) for i, w in bad))


JPEG_ERRORS = {1: "invalid Huffman code", 2: "entropy-coded data ends early", 4: "restart marker out of sequence"}


def decode_png_batch(files: Sequence, stream: Optional[torch.cuda.Stream] = None, with_status: bool = False):
    """GPU-decodable PNG files (``bytes``, ``bytearray``, ``memoryview``) -> list of CUDA uint8 [h, w, 3] RGB views of one
    packed device buffer, byte for byte what ``Helper._read_img`` (PIL) gives.  One pinned staging buffer, one H2D copy and
    one launch per decode stage on `stream` (default: the current stream), then a synchronise to read the per-image status.
    A file the GPU decoder does not take raises ``ValueError`` before anything is enqueued; a zlib stream PIL refuses raises
    ``K2YError`` naming the images, unless `with_status`, which returns (views, status int32 [n, 4]: error bits, chunks, chunks
    whose speculative start was confirmed, bytes the longest single decoder inflated) instead."""
    if not isinstance(files, (list, tuple)) or len(files) == 0:
        raise ValueError("expected a non-empty list of PNG files")
    bufs, shapes = [], []
    for i, f in enumerate(files):
        if not isinstance(f, ENCODED):
            raise ValueError(f"file {i}: expected bytes, bytearray or memoryview, got {type(f).__name__}")
        buf = _file_bytes(f)
        if _png_route(buf) is None:
            info = _png_info(buf)
            why = "not a PNG file with a sound IHDR" if info is None else inspect_png(f)[3]
            raise ValueError(f"file {i}: not decodable on the GPU: {why}")
        info = _png_info(buf)
        bufs.append(buf)
        shapes.append((int(info.height), int(info.width)))
    sizes = np.array([h * w * 3 for h, w in shapes], np.int64)
    padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
    offsets = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    device = torch.device("cuda", torch.cuda.current_device())
    st = stream if stream is not None else torch.cuda.current_stream(device)
    staging = Staging(device, st)
    plan = _jpeg_layout(bufs, offsets, int(padded.sum()), _png_plan)
    staging.reserve(plan[3], len(bufs))
    with torch.cuda.stream(st):
        stage_pngs(bufs, offsets, staging, plan, staging.dev)
        status = staging.png_status[:len(bufs)].cpu().numpy()
    out = [staging.dev[o:o + h * w * 3].view(h, w, 3) for o, (h, w) in zip(offsets, shapes)]
    if with_status:
        return out, status
    check_png_status(status, range(len(bufs)))
    return out


PNG_ERRORS = {1: "invalid block header", 2: "invalid code", 4: "distance too far back", 8: "image data ends early",
              16: "Adler-32 mismatch", 32: "filter type above 4"}


def check_png_status(status: np.ndarray, images) -> None:
    """Raises ``K2YError`` naming the images whose zlib stream or row filters PIL refuses.  `status`: the decode's int32 [n, 4]
    words of the GPU-decoded PNGs, `images`: their positions in the caller's batch."""
    bad = [(int(i), int(w)) for i, w in zip(images, status[:, 0]) if w]
    if bad:
        raise K2YError("corrupt PNG data: " + ", ".join(
            f"image {i}: " + ", ".join(v for k, v in PNG_ERRORS.items() if w & k) for i, w in bad))


def decode_progressive_jpeg_batch(files: Sequence, stream: Optional[torch.cuda.Stream] = None, with_status: bool = False):
    """GPU-decodable progressive JPEG files (``bytes``, ``bytearray``, ``memoryview``) -> list of CUDA uint8 [h, w, 3] RGB views
    of one packed device buffer, byte for byte what ``Helper._read_img`` (PIL) gives.  One pinned staging buffer, one H2D copy,
    one entropy-decode launch per level of the scan scripts and one IDCT and one colour launch on `stream` (default: the
    current stream), then a synchronise to read the per-image status.  A file the GPU decoder does not take raises
    ``ValueError`` before anything is enqueued; corrupt entropy data raises ``K2YError`` naming the images, unless
    `with_status`, which returns (views, status int32 [n, 4]: error bits, 0, 0, segments decoded) instead."""
    if not isinstance(files, (list, tuple)) or len(files) == 0:
        raise ValueError("expected a non-empty list of progressive JPEG files")
    bufs, shapes = [], []
    for i, f in enumerate(files):
        if not isinstance(f, ENCODED):
            raise ValueError(f"file {i}: expected bytes, bytearray or memoryview, got {type(f).__name__}")
        buf = _file_bytes(f)
        info = _progressive_info(buf)
        if info is None or not info.gpu_decodable:
            why = info.reason.decode() if info is not None else "not a well-formed JPEG file"
            raise ValueError(f"file {i}: not decodable on the GPU: {why}")
        bufs.append(buf)
        shapes.append((int(info.height), int(info.width)))
    sizes = np.array([h * w * 3 for h, w in shapes], np.int64)
    padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
    offsets = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    device = torch.device("cuda", torch.cuda.current_device())
    st = stream if stream is not None else torch.cuda.current_stream(device)
    staging = Staging(device, st)
    plan = _jpeg_layout(bufs, offsets, int(padded.sum()), _progressive_plan)
    staging.reserve(plan[3], len(bufs))
    with torch.cuda.stream(st):
        stage_progressive_jpegs(bufs, offsets, staging, plan, staging.dev)
        status = staging.progressive_status[:len(bufs)].cpu().numpy()
    out = [staging.dev[o:o + h * w * 3].view(h, w, 3) for o, (h, w) in zip(offsets, shapes)]
    if with_status:
        return out, status
    check_progressive_status(status, range(len(bufs)))
    return out


PROGRESSIVE_ERRORS = {1: "invalid Huffman code", 2: "entropy-coded data ends early", 4: "DC value out of range"}


def check_progressive_status(status: np.ndarray, images) -> None:
    """Raises ``K2YError`` naming the progressive JPEGs whose entropy-coded data was corrupt or ended early.  `status`: the
    decode's int32 [n, 4] words of the GPU-decoded progressive JPEGs, `images`: their positions in the caller's batch."""
    bad = [(int(i), int(w)) for i, w in zip(images, status[:, 0]) if w]
    if bad:
        raise K2YError("corrupt progressive JPEG data: " + ", ".join(
            f"image {i}: " + ", ".join(v for k, v in PROGRESSIVE_ERRORS.items() if w & k) for i, w in bad))
