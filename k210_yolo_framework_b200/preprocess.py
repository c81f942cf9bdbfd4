"""GPU pre-processing mirror of ``Helper._process_img`` (tools/utils.py:357-406, inference branch).

``letterbox_params`` builds the affine parameters exactly as the reference does (numpy, a handful of host flops);
``letterbox_device`` runs the resampling on the GPU through the C-ABI (``k2y_letterbox_u8``, csrc/preprocess.cu) and
returns the uint8 network input; the ``img / np.max(img)`` normalisation is fused into the network's uint8 front end
(``YoloEngine.predict_device_u8``).  There is no CPU fallback: without the CUDA library the call raises.

``letterbox_batch_device`` does the same for a list of host images of different sizes in one launch: ``BatchLayout`` packs
them back to back into one pinned staging buffer (``Staging``), one H2D copy moves the whole batch and
``k2y_letterbox_u8_batch`` letterboxes every image into one uint8 [n, in_h, in_w, 3] tensor.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import numpy as np
import torch

from ._lib import check, lib


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


def _check_images(images) -> None:
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("expected a non-empty list of host uint8 [h, w, 3] arrays")
    for i, im in enumerate(images):
        if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
            desc = f"{im.dtype} {im.shape}" if isinstance(im, np.ndarray) else type(im).__name__
            raise ValueError(f"image {i}: expected a host numpy uint8 [h, w, 3] array, got {desc}")


class BatchLayout:
    """Where each image of a ragged batch lies in the packed buffer, and its letterbox descriptor.

    ``offsets`` int64 [n] (multiples of ``ALIGN``), ``hw`` int32 [n, 2] (h, w), ``matrices`` float64 [n, 6] (the first two
    rows of ``letterbox_params``' inverse matrix), ``nbytes`` the packed size."""

    def __init__(self, images: Sequence[np.ndarray], in_hw):
        _check_images(images)
        n = len(images)
        self.in_hw = (int(in_hw[0]), int(in_hw[1]))
        self.hw = np.array([im.shape[:2] for im in images], dtype=np.int32).reshape(n, 2)
        sizes = self.hw[:, 0].astype(np.int64) * self.hw[:, 1] * 3
        padded = (sizes + ALIGN - 1) // ALIGN * ALIGN
        self.offsets = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
        self.nbytes = int(padded.sum())
        self.matrices = np.array([letterbox_params((int(h[0]), int(h[1])), self.in_hw)[2][:2].reshape(-1) for h in self.hw], dtype=np.float64)

    def __len__(self) -> int:
        return len(self.hw)

    def pack(self, images: Sequence[np.ndarray], host: np.ndarray) -> None:
        """Copies `images` into the uint8 buffer `host` (at least ``nbytes`` long) at their offsets."""
        for im, off, (h, w) in zip(images, self.offsets, self.hw):
            np.copyto(host[off:off + h * w * 3].reshape(h, w, 3), im)


class Staging:
    """A pinned host buffer and a device buffer for packed batches, plus the kernel's min/max scratch, reused across calls.
    They grow (geometrically) only when a batch does not fit; the caller makes sure the previous H2D copy out of the host
    buffer has finished first.  The device buffers are allocated on `stream`, the stream that reads them."""

    def __init__(self, device: torch.device, stream: torch.cuda.Stream):
        self.device, self.stream = device, stream
        self.host: Optional[torch.Tensor] = None
        self.dev: Optional[torch.Tensor] = None
        self.minmax: Optional[torch.Tensor] = None

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


def letterbox_packed(layout: BatchLayout, images: Sequence[np.ndarray], staging: Staging, out: torch.Tensor,
                     image_hw_out: Optional[torch.Tensor]) -> None:
    """Packs `images` into ``staging.host``, copies them to the device and letterboxes them into ``out[:n]`` (and their sizes
    into ``image_hw_out[:n]``), all on ``staging.stream``.  The host buffer is reused by the next call: wait for this copy
    before packing into it again."""
    n = len(layout)
    staging.reserve(layout.nbytes, n)
    layout.pack(images, staging.host.numpy())
    in_h, in_w = layout.in_hw
    st = staging.stream
    with torch.cuda.stream(st):
        staging.dev[:layout.nbytes].copy_(staging.host[:layout.nbytes], non_blocking=True)
        offs = layout.offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong))
        hw = layout.hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
        mats = layout.matrices.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        check(lib.k2y_letterbox_u8_batch(staging.dev.data_ptr(), n, offs, hw, mats, out.data_ptr(), in_h, in_w,
                                         image_hw_out.data_ptr() if image_hw_out is not None else None, staging.minmax.data_ptr(),
                                         ctypes.c_void_p(st.cuda_stream)))


def letterbox_batch_device(images: List[np.ndarray], in_hw, out: Optional[torch.Tensor] = None,
                           image_hw_out: Optional[torch.Tensor] = None, stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
    """images: host numpy uint8 [h, w, 3] RGB arrays of any sizes -> CUDA uint8 [n, in_h, in_w, 3] letterboxed (zero fill), the
    same bytes ``letterbox_device`` gives each image.  One pinned staging buffer, one H2D copy, one batched letterbox launch on
    `stream` (default: the current stream), asynchronous.  `out` ([N >= n, in_h, in_w, 3] uint8, e.g. a network's bound input)
    receives the images in its first n rows; `image_hw_out` ([N >= n, 2] float32), if given, receives each image's (h, w)."""
    in_h, in_w = int(in_hw[0]), int(in_hw[1])
    layout = BatchLayout(images, (in_h, in_w))
    n = len(layout)
    device = out.device if out is not None else torch.device("cuda", torch.cuda.current_device())
    _check_out(out, n, (in_h, in_w, 3), torch.uint8, "out", None)
    _check_out(image_hw_out, n, (2,), torch.float32, "image_hw_out", device)
    st = stream if stream is not None else torch.cuda.current_stream(device)
    if out is None:
        with torch.cuda.stream(st):
            out = torch.empty((n, in_h, in_w, 3), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        letterbox_packed(layout, images, Staging(device, st), out, image_hw_out)
    return out
