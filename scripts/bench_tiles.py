#!/usr/bin/env python
"""Tiled detection on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32): what detecting on 2x2 or 3x3 overlapping tiles beside the
whole image costs, on the bench_ingest photos as decoded pixels and as quality-90 JPEG bytes.

  * images/s of ``submit_images`` / ``collect`` (two batches in flight) with tiling off, 2x2 and 3x3, per route, and the network
    inputs/s that is (images/s x views per image).  One pipeline per tiling, all warmed up first, timed in alternating windows
    (median of --windows); every window ends in a device synchronise.
  * kernel time of the views letterbox (``k2y_letterbox_u8_views``: one memset and two kernels per call, on a batch already on
    the device) and of the merge (``k2y_merge_views``), CUDA events around --launches calls each.
  * one check that the tiled records equal the composed reference: the crops through the untiled pipeline, then the numpy merge
    of oracle/tiles_ref.py.
  * with --tile_size H W --tile_images N, one more arm ("size"): each image cut into tiles of at most H x W pixels
    (``enable_tiling(tile_size=..., images_per_batch=N)``), timed like the others, checked against oracle/tiles_merge_ref.py,
    and ``k2y_merge_views_ex`` timed on one of its batches in every metric / action mode, and with a border.
  * with --flip, two more arms: "flip" (every image and its mirror, ``enable_flip``) and "2x2+flip" (2x2 tiles and the whole
    image, each also mirrored), timed like the others, checked against the composed reference of oracle/flip_ref.py
    (the crops and their np.fliplr through the untiled pipeline, then the merge with the mirror flags), and the mirrored
    letterbox (``k2y_letterbox_u8_views_mirror``) and merge (``k2y_merge_views_mirror``) timed on one of their batches.

The card's name, power limit and SM clock are read in the same run.  Prints one JSON line.

    python scripts/bench_tiles.py [--images 192 --batch 32 --windows 3 --passes 4 --launches 200 --tile_size 224 320
                                   --tile_images 6 --flip]
"""
import argparse
import ctypes
import io
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_ingest import GOLDEN, gpu_info, photos  # noqa: E402
from k210_yolo_framework_b200 import preprocess, tiles  # noqa: E402
from k210_yolo_framework_b200._lib import check, lib  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.yolonet import load_npz_weights  # noqa: E402

TILINGS = {"off": None, "2x2": (2, 2), "3x3": (3, 3)}
NBOX = 1050


def run(pipe, images):
    """All `images` through submit_images / collect, two batches in flight; returns the records per image."""
    B = pipe.images_per_batch
    recs, pending = [], []
    for i in range(0, len(images), B):
        pending.append(pipe.submit_images(images[i:i + B]))
        if len(pending) == 2:
            recs += DetectionPipeline.records(*pipe.collect(pending.pop(0)))
    for t in pending:
        recs += DetectionPipeline.records(*pipe.collect(t))
    return recs


def composed_sized(plain, images, tile_hw, images_per_batch, cap, overlap, iou):
    """The crops of every planned view through the untiled pipeline, one tiled batch's views per batch, then the numpy merge."""
    from oracle import tiles_merge_ref as ref
    out = []
    for i in range(0, len(images), images_per_batch):
        chunk = images[i:i + images_per_batch]
        per = [ref.plan_windows(im.shape[0], im.shape[1], tile_hw, overlap, cap) for im in chunk]
        windows = np.concatenate(per)
        offsets = np.concatenate([[0], np.cumsum([len(w) for w in per])])
        crops = [np.ascontiguousarray(im[y0:y0 + th, x0:x0 + tw]) for im, w in zip(chunk, per) for y0, x0, th, tw in w.tolist()]
        d, c = plain.collect(plain.submit_images(crops))
        dets, counts = ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], offsets, NBOX, iou)
        out += [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
                 for cls in range(dets.shape[1]) for r in dets[b, cls, :counts[b, cls]]] for b in range(len(chunk))]
    return out


def composed(plain, images, rows, cols, overlap, iou):
    """The crops of every view through the untiled pipeline, one tiled batch's views per batch, then the numpy merge."""
    from oracle import tiles_ref
    V = 1 + rows * cols
    per = plain.batch // V
    out = []
    for i in range(0, len(images), per):
        chunk = images[i:i + per]
        windows = np.concatenate([tiles_ref.tile_windows(im.shape[0], im.shape[1], rows, cols, overlap) for im in chunk])
        crops = [np.ascontiguousarray(chunk[j // V][y0:y0 + th, x0:x0 + tw]) for j, (y0, x0, th, tw) in enumerate(windows.tolist())]
        d, c = plain.collect(plain.submit_images(crops))
        dets, counts = tiles_ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], len(chunk), NBOX, iou)
        out += [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
                 for cls in range(dets.shape[1]) for r in dets[b, cls, :counts[b, cls]]] for b in range(len(chunk))]
    return out


def composed_flip(plain, images, images_per_batch, rows_cols, overlap, iou):
    """The crops of every view and their mirrors through the untiled pipeline, one flipped batch's views per batch, then the
    numpy merge with the mirror flags."""
    from oracle import flip_ref
    out = []
    for i in range(0, len(images), images_per_batch):
        chunk = images[i:i + images_per_batch]
        per = [tiles.tile_windows(im.shape[0], im.shape[1], *rows_cols, overlap) if rows_cols else
               np.array([(0, 0, im.shape[0], im.shape[1])], np.int32) for im in chunk]
        crops, windows, mirror = [], [], []
        for im, w in zip(chunk, per):
            cut = [np.ascontiguousarray(im[y0:y0 + th, x0:x0 + tw]) for y0, x0, th, tw in w.tolist()]
            crops += cut + [np.ascontiguousarray(np.fliplr(c)) for c in cut]
            windows += [w, w]
            mirror += [0] * len(w) + [1] * len(w)
        windows = np.concatenate(windows)
        offsets = np.concatenate([[0], np.cumsum([2 * len(w) for w in per])])
        d, c = plain.collect(plain.submit_images(crops))
        dets, counts = flip_ref.merge_views(d.numpy(), c.numpy(), windows[:, :2], offsets, NBOX, iou, view_hw=windows[:, 2:],
                                       mirrored=np.array(mirror))
        out += [[(cls, int(r["index"]), float(r["score"]), float(r["ymin"]), float(r["xmin"]), float(r["ymax"]), float(r["xmax"]))
                 for cls in range(dets.shape[1]) for r in dets[b, cls, :counts[b, cls]]] for b in range(len(chunk))]
    return out


def events_ms(fn, launches):
    """Milliseconds per call of `fn` over `launches` calls on the current stream, after 10 warm-up calls."""
    for _ in range(10):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / launches


def kernel_times(pipe, images, launches):
    """(views letterbox ms, merge ms, views) for one full tiled batch of `pipe`, its inputs resident on the device.  For a
    pipeline tiled by size the merge time is a dict: ``k2y_merge_views_ex`` in every metric / action mode, and with a border."""
    imgs = images[:pipe.images_per_batch]
    sized = pipe._merge is not None
    flip = pipe._flip
    layout = preprocess.BatchLayout(imgs, pipe.in_hw, pipe._tiling, merge_table=sized, flip=flip)
    n, N, V = len(layout), layout.n_views, pipe._views
    dev = torch.device("cuda", pipe.device_index)
    st = torch.cuda.current_stream()
    staging = preprocess.Staging(dev, st)
    out = torch.empty((N,) + pipe.in_hw + (3,), dtype=torch.uint8, device=dev)
    hw = torch.empty((N, 2), device=dev)
    yx = torch.empty((N, 2), device=dev)
    preprocess.letterbox_packed(layout, imgs, staging, out, hw, yx)     # packs and copies the batch; the loop below only letterboxes
    offsets = np.repeat(layout.offsets, layout.view_counts)
    full = np.ascontiguousarray(np.repeat(layout.hw, layout.view_counts, axis=0))

    def letterbox_mirror():
        check(lib.k2y_letterbox_u8_views_mirror(
            staging.dev.data_ptr(), N, offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
            full.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), layout.windows.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
            layout.view_mirror.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
            layout.view_matrices.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), out.data_ptr(), pipe.in_hw[0], pipe.in_hw[1],
            hw.data_ptr(), yx.data_ptr(), staging.minmax.data_ptr(), ctypes.c_void_p(st.cuda_stream)))

    def letterbox():
        check(lib.k2y_letterbox_u8_views(staging.dev.data_ptr(), N, offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                         full.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                         layout.windows.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                         layout.view_matrices.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), out.data_ptr(),
                                         pipe.in_hw[0], pipe.in_hw[1], hw.data_ptr(), yx.data_ptr(), staging.minmax.data_ptr(),
                                         ctypes.c_void_p(st.cuda_stream)))

    # the per-view block of the batch the pipeline ran last is still in place: merge it again into a scratch gather slot
    pipe.collect(pipe.submit_images(imgs))
    torch.cuda.synchronize()
    slot = torch.empty_like(pipe.gather.bufs[0])
    dets, counts = pipe.gather.split(slot, pipe.gather.C, pipe.gather.K)

    def merge():
        check(lib.k2y_merge_views(pipe._view_dets.data_ptr(), pipe._view_counts.data_ptr(), yx.data_ptr(), n, pipe.batch, V, NBOX,
                                  pipe.gather.C, pipe.gather.K, pipe.detector.cfg.iou_thresh, dets.data_ptr(), counts.data_ptr(),
                                  dets.stride(0), counts.stride(0), ctypes.c_void_p(st.cuda_stream)))

    def merge_ex(match, merge, border):
        table = staging.dev.data_ptr() + layout.merge_table_at
        return lambda: check(lib.k2y_merge_views_ex(
            pipe._view_dets.data_ptr(), pipe._view_counts.data_ptr(), yx.data_ptr(), table, table + 4 * (n + 1) if border else None,
            hw.data_ptr() if border else None, border if border else -1.0, match, merge, n, pipe.batch, V, NBOX, pipe.gather.C,
            pipe.gather.K, pipe.detector.cfg.iou_thresh, dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0),
            ctypes.c_void_p(st.cuda_stream)))

    def merge_mirror():
        table = staging.dev.data_ptr() + layout.merge_table_at
        check(lib.k2y_merge_views_mirror(
            pipe._view_dets.data_ptr(), pipe._view_counts.data_ptr(), yx.data_ptr(), table, None, table + 4 * (n + 1 + N),
            hw.data_ptr(), -1.0, 0, 0, n, pipe.batch, V, NBOX, pipe.gather.C, pipe.gather.K, pipe.detector.cfg.iou_thresh,
            dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0), ctypes.c_void_p(st.cuda_stream)))

    if flip:
        return events_ms(letterbox_mirror, launches), events_ms(merge_mirror, launches), N
    if not sized:
        return events_ms(letterbox, launches), events_ms(merge, launches), N
    modes = {f"{m}/{a}": (i, j, None) for i, m in enumerate(("iou", "ios")) for j, a in enumerate(("suppress", "union"))}
    modes["ios/union/border2"] = (1, 1, 2.0)
    return events_ms(letterbox, launches), {k: round(events_ms(merge_ex(*v), launches), 4) for k, v in modes.items()}, N


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=192, help="a multiple of 96, so that every tiling runs full batches")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--passes", type=int, default=4, help="passes over the images per window")
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--obj_thresh", type=float, default=0.3)
    ap.add_argument("--tile_size", type=int, nargs=2, default=None, metavar=("H", "W"), help="add an arm tiled by tile size")
    ap.add_argument("--tile_images", type=int, default=6, help="images per batch of the --tile_size arm")
    ap.add_argument("--flip", action="store_true", help="add the arms flip (each image and its mirror) and 2x2+flip")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tiles measures on a GPU"
    from PIL import Image
    torch.cuda.set_device(0)
    H, W = 224, 320
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    weights = load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz"))
    pipes = {}
    tilings = dict(TILINGS)
    if args.tile_size:
        tilings["size"] = "size"
    if args.flip:
        tilings["flip"], tilings["2x2+flip"] = "flip", (2, 2, "flip")
    for name, t in tilings.items():
        pipes[name] = DetectionPipeline("yolo_mobilev1", (H, W), anchors, 20, 0.75, args.batch, obj_thresh=args.obj_thresh, iou_thresh=0.5)
        pipes[name].engine.set_weights(weights)
        if t == "size":
            pipes[name].enable_tiling(tile_size=tuple(args.tile_size), images_per_batch=args.tile_images)
        elif t == "flip":
            pipes[name].enable_flip()
        elif t:
            pipes[name].enable_tiling(*t[:2])
            if t[2:] == ("flip",):
                pipes[name].enable_flip()
    pixels = photos(args.images)
    files = []
    for img in pixels:
        f = io.BytesIO()
        Image.fromarray(img).save(f, "JPEG", quality=90)
        files.append(f.getvalue())
    routes = {"pixels": pixels, "jpeg": files}

    # warm-up of every pipeline on both routes; the check uses the pixel route of the first 24 images
    first = {(name, r): run(pipes[name], imgs) for name in tilings for r, imgs in routes.items()}
    equal = {}
    for name in ("2x2", "3x3"):
        rows, cols = TILINGS[name]
        k = 8 * pipes[name].images_per_batch
        equal[name] = first[(name, "pixels")][:k] == composed(pipes["off"], pixels[:k], rows, cols, 0.2, 0.5)
    views_per_image = {n: 1 + t[0] * t[1] if t else 1 for n, t in TILINGS.items()}
    if args.tile_size:
        p = pipes["size"]
        k = 8 * p.images_per_batch
        equal["size"] = first[("size", "pixels")][:k] == composed_sized(pipes["off"], pixels[:k], tuple(args.tile_size),
                                                                         p.images_per_batch, p._views, 0.2, 0.5)
        views_per_image["size"] = float(np.mean([len(tiles.plan_windows(im.shape[0], im.shape[1], tuple(args.tile_size), 0.2, p._views))
                                                 for im in pixels]))
    if args.flip:
        for name, rc in (("flip", None), ("2x2+flip", (2, 2))):
            p = pipes[name]
            k = 4 * p.images_per_batch
            equal[name] = first[(name, "pixels")][:k] == composed_flip(pipes["off"], pixels[:k], p.images_per_batch, rc, 0.2, 0.5)
            views_per_image[name] = p._views
    records = {f"{name}/{r}": sum(len(x) for x in v) for (name, r), v in first.items()}

    times = {k: [] for k in first}
    for _ in range(args.windows):
        for (name, r) in times:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.passes):
                run(pipes[name], routes[r])
            torch.cuda.synchronize()
            times[(name, r)].append(time.perf_counter() - t0)
    rate = {k: args.passes * len(pixels) / statistics.median(v) for k, v in times.items()}
    kernels = {}
    for name in [n for n in tilings if n != "off"]:
        lb, mg, nv = kernel_times(pipes[name], pixels, args.launches)
        kernels[name] = {"views": nv, "letterbox_views_ms": round(lb, 4), "merge_views_ms": mg if isinstance(mg, dict) else round(mg, 4)}
    print(json.dumps({
        "metric": "tiled_img_per_s", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}, obj_thresh {args.obj_thresh}",
        "images": len(pixels), "passes": args.passes,
        "images_per_s": {f"{n}/{r}": round(v, 1) for (n, r), v in rate.items()},
        "network_inputs_per_s": {f"{n}/{r}": round(v * views_per_image[n], 1) for (n, r), v in rate.items()},
        "views_per_image": views_per_image, "tile_size": args.tile_size, "tile_images": args.tile_images if args.tile_size else None,
        "windows_s": {f"{n}/{r}": [round(t, 4) for t in v] for (n, r), v in times.items()},
        "flip": args.flip, "records": records, "kernels": kernels, "launches": args.launches, "equals_composed_reference": equal, "gpu": gpu_info()}))
    if not all(equal.values()):
        sys.exit("tiled records differ from the composed reference")


if __name__ == "__main__":
    main()
