"""Inference-side mirror of ``tools.utils.Helper`` (/root/reference/tools/utils.py:53-82, 233-271, 339-406).

Holds what ``keras_inference.py:main`` takes from the helper: ``in_hw``, ``out_hw``, ``anchors`` ([L,A,2]
(w,h) as a fraction of the network input, loaded from ``data/{train_set}_anchor.npy``), ``class_num``,
``colormap``; plus ``_read_img`` / ``_process_img`` (aspect-preserving letterbox, zero fill, ``img/np.max(img)``).
The training-side members (dataset lists, augmenter, label encoding, loss helpers) are out of scope.
"""
from __future__ import annotations

import numpy as np


class Helper(object):
    def __init__(self, image_ann, class_num: int, anchors, in_hw, out_hw, validation_split=0.1):
        self.in_hw = np.array(in_hw)
        assert self.in_hw.ndim == 2
        self.out_hw = np.array(out_hw)
        assert self.out_hw.ndim == 2
        if image_ann is not None:
            raise NotImplementedError("training data lists are out of scope for the inference path")
        self.grid_wh = (1 / self.out_hw)[:, [1, 0]]
        self.class_num = class_num
        self.anchors = np.load(anchors) if isinstance(anchors, (str, bytes)) or hasattr(anchors, "__fspath__") \
            else np.asarray(anchors)
        self.anchor_number = len(self.anchors[0])
        self.output_number = len(self.anchors)
        if self.output_number != len(self.out_hw):
            raise ValueError(f"anchor file has {self.output_number} layers, output_size gives {len(self.out_hw)}")
        self.colormap = _COLORMAP

    def _read_img(self, img_path: str) -> np.ndarray:
        """tools/utils.py:339-355 (skimage.io.imread -> RGB uint8, grey -> 3 channels, alpha dropped)."""
        return read_image(img_path)

    def _process_img(self, img: np.ndarray, true_box=None, is_training: bool = False, is_resize: bool = True):
        """tools/utils.py:357-406, inference branch: letterbox to in_hw[0] then ``img / np.max(img)``.

        The resampling runs on the GPU (``preprocess.letterbox_device`` -> k2y_letterbox_u8): the affine parameters follow the
        reference exactly (scale = min(in_wh/img_wh), translation = ((in_wh - img_wh*scale)/2).astype(int)) and the
        interpolation restates skimage 0.15's ``warp`` (order 1, zero fill, clip, uint8 truncation; third-party, not
        available offline — oracle/preprocess_ref.py).  Exact for an image that already has the network size.
        Returns the reference's value: a float64 HxWx3 array in [0, 1] on the host.
        """
        if is_training:
            raise NotImplementedError("augmentation is out of scope for the inference path")
        if is_resize:
            img = self.letterbox_device(img).cpu().numpy()
        img = img / np.max(img)
        return img, true_box

    def letterbox_device(self, img: np.ndarray):
        """uint8 HWC host image -> CUDA uint8 [in_h, in_w, 3]: the input of the network's uint8 front end
        (``predict_device_u8``), which applies ``img / np.max(img)`` on the GPU."""
        import torch
        from .preprocess import letterbox_device
        x = torch.from_numpy(np.array(img[..., :3], dtype=np.uint8, order="C", copy=True)).cuda()
        return letterbox_device(x, self.in_hw[0])


# Helper.colormap (tools/utils.py:89-105): 80 RGB triples, one per class id, kept as packed bytes (r,g,b,r,g,b,...)
_COLORMAP_RGB = bytes.fromhex(
    "ff520000fff5003dff00ff7000ff85ff0000ffa300ff6600c2ff00008fff33ff000052ff00ff2900ffad0a00ffadff00"
    "00ff99ff5c00ff00ffff00f5800000008000808000000080800080008080808080400000c00000408000c08000400080"
    "c00080408080c0808000400080400000c00080c0000040803de6faff06330b66ffff0747ff09e00907e6dcdcdcff095c"
    "7009ff08ffd607ffe0ffb8060aff47ff290a07ffffe0ff086608ffff3d06ffc207ff7a0800ff14ff0829ff05990633ff"
    "eb0cffa0961400a3ff8c8c8cfa0a0f14ff001fff00ff1f00ffe00099ff000000ffff470000ebff00adff1f00ff0bc8c8")
_COLORMAP = [tuple(_COLORMAP_RGB[i:i + 3]) for i in range(0, len(_COLORMAP_RGB), 3)]


def read_image(img_path) -> np.ndarray:
    """``Helper._read_img``: `img_path` is a path or a binary file object (e.g. ``io.BytesIO`` of a file's bytes)."""
    from PIL import Image
    im = Image.open(img_path)
    # skimage.io.imread semantics by PIL mode: palette / CMYK / YCbCr images are expanded to RGB, grey (+alpha) becomes
    # 3 equal channels, 16/32-bit grey is scaled down to 8 bits, alpha is dropped
    if im.mode in ("P", "CMYK", "YCbCr", "PA"):
        im = im.convert("RGB")
    elif im.mode in ("LA", "La"):
        im = im.convert("L")
    elif im.mode == "1":
        im = im.convert("L")
    elif im.mode in ("I", "I;16", "I;16B", "I;16L", "F"):
        arr = np.asarray(im, dtype=np.float64)
        hi = float(arr.max()) if arr.size else 0.0
        im = Image.fromarray(np.clip(arr * (255.0 / hi if hi > 255.0 else 1.0), 0, 255).astype(np.uint8))
    elif im.mode not in ("RGB", "RGBA", "L"):
        im = im.convert("RGB")
    img = np.asarray(im, dtype=np.uint8)
    if img.ndim != 3:
        img = np.stack([img] * 3, axis=-1)
    return img[..., :3]
