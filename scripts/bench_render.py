#!/usr/bin/env python
"""Drawn results on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32), one process, one GPU.  The images are bench_ingest's seeded
photos (five sizes, 375x500 to 720x1280) as JPEG files in memory (PIL, quality 90, 4:2:0), the records come from the golden
VOC weights at obj_thresh 0.3.  Reports:

  kernels:      render + encode of one batch of 32 decoded images with their records (k2y_render_detections + the seven
                k2y_jpeg_encode launches), CUDA events over many batches, and each kernel's device time from torch.profiler;
  files/s:      file bytes -> records + drawn JPEG files through DetectionPipeline.submit_images(bytes) + rendered() (two
                batches in flight), against the same submit_images(bytes) + collect followed by PIL draw_detections + save
                in 1, 4 and 16 host threads; alternating windows, median of three;
  files_equal:  every route gives the same bytes (the run fails otherwise);

and the card's name, power limit and SM clock, read in the same run.  Prints one JSON line.

    python scripts/bench_render.py [--images 256 --batch 32 --windows 3 --passes 2 --quality 75 --reps 30]
"""
import argparse
import io
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_decode import jpeg_files  # noqa: E402
from bench_ingest import GOLDEN, SIZES, gpu_info, photos  # noqa: E402
from k210_yolo_framework_b200 import preprocess  # noqa: E402
from k210_yolo_framework_b200.draw import draw_detections  # noqa: E402
from k210_yolo_framework_b200.helper import _COLORMAP, read_image  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.render import JpegEncoder, LabelAtlas, color_table, render_packed  # noqa: E402
from k210_yolo_framework_b200.yolonet import load_npz_weights  # noqa: E402

KERNELS = ("render_kernel", "enc_dct_kernel", "enc_len_kernel", "enc_scan_kernel", "enc_emit_kernel", "enc_ffcount_kernel",
           "enc_ffscan_kernel", "enc_pack_kernel")


def run_gpu(pipe, batches):
    out, pending = [], []
    for files in batches:
        pending.append(pipe.submit_images(files))
        if len(pending) == 2:
            t = pending.pop(0)
            pipe.collect(t)
            out.extend(pipe.rendered(t))
    for t in pending:
        pipe.collect(t)
        out.extend(pipe.rendered(t))
    return out


def pil_file(data, recs, quality):
    b = io.BytesIO()
    draw_detections(read_image(io.BytesIO(data)), recs, _COLORMAP).save(b, "JPEG", quality=quality)
    return b.getvalue()


def run_pil(pipe, batches, pool, quality):
    out, pending = [], []

    def finish(t, files):
        recs = DetectionPipeline.records(*pipe.collect(t))
        out.extend(pool.map(pil_file, files, recs, [quality] * len(files)))
    for files in batches:
        pending.append((pipe.submit_images(files), files))
        if len(pending) == 2:
            finish(*pending.pop(0))
    for p in pending:
        finish(*p)
    return out


def time_kernels(pipe, files, quality, reps):
    """Device ms of render + encode of one batch (events around `reps` calls) and per kernel (torch.profiler)."""
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev)
    views = preprocess.decode_jpeg_batch(files)
    t = pipe.submit_images(files)
    pipe.collect(t)
    dets, counts = pipe.gather.local(t)
    base = min(v.data_ptr() for v in views)
    offsets = np.array([v.data_ptr() - base for v in views], np.int64)
    hw = np.array([v.shape[:2] for v in views], np.int32)
    atlas, colors, enc = LabelAtlas(20), color_table(_COLORMAP, 20, dev), JpegEncoder(dev)

    def once():
        render_packed(base, offsets, hw, dets[:len(files)], counts[:len(files)], atlas, colors, dev, st)
        enc.enqueue(base, offsets, hw, quality, st)
    for _ in range(3):
        once()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(st)
    for _ in range(reps):
        once()
    t1.record(st)
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    from torch.profiler import ProfilerActivity, profile
    prof_reps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(prof_reps):
            once()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                kernels[k] = kernels.get(k, 0.0) + e.device_time_total / 1e3 / prof_reps
    return ms, kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--passes", type=int, default=2, help="passes over the images per window")
    ap.add_argument("--quality", type=int, default=75)
    ap.add_argument("--reps", type=int, default=30, help="render + encode calls timed per batch")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_render measures on a GPU"
    torch.cuda.set_device(0)
    files = jpeg_files(photos(args.images))
    batches = [files[i:i + args.batch] for i in range(0, len(files), args.batch)]
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, args.batch, obj_thresh=0.3, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))

    # (1) the kernels, per batch
    ms, kernel_ms = [], {}
    for b in batches:
        t, kern = time_kernels(pipe, b, args.quality, args.reps)
        ms.append(t)
        for k, v in kern.items():
            kernel_ms[k] = kernel_ms.get(k, 0.0) + v / len(batches)
    per_batch = statistics.mean(ms)

    # (2) files/s from file bytes to drawn JPEG files
    gpu = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, args.batch, obj_thresh=0.3, iou_thresh=0.5)
    gpu.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    gpu.enable_rendering(quality=args.quality)
    threads = (1, 4, 16)
    pools = {k: ThreadPoolExecutor(k) for k in threads}
    routes = {"gpu_render": lambda: run_gpu(gpu, batches)}
    for k in threads:
        routes[f"pil_{k}_threads"] = (lambda k=k: run_pil(pipe, batches, pools[k], args.quality))
    ref = routes["gpu_render"]()
    same = all(fn() == ref for fn in routes.values())       # warm-up of every route, and the equality check
    times = {k: [] for k in routes}
    for _ in range(args.windows):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = [fn() for _ in range(args.passes)]
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            same = same and all(r == ref for r in out)
    for p in pools.values():
        p.shutdown()
    rate = {k: round(args.passes * len(files) / statistics.median(v), 1) for k, v in times.items()}
    print(json.dumps({
        "metric": "render_encode", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}, obj_thresh 0.3", "images": len(files),
        "sizes": [list(s) for s in SIZES], "input": "PIL quality 90, 4:2:0", "quality": args.quality,
        "records_per_image": round(sum(len(r) for b in batches for r in DetectionPipeline.records(*gpu.collect(gpu.submit_images(b)))) / len(files), 2),
        "render_encode_ms_per_batch": round(per_batch, 4), "render_encode_img_per_s": round(args.batch / per_batch * 1e3, 1),
        "kernel_ms_per_batch": {k: round(v, 4) for k, v in kernel_ms.items()},
        "files_per_s": rate, "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()}, "files_equal": same,
        "mean_file_kb": round(sum(len(f) for f in ref) / len(ref) / 1e3, 2), "gpu": gpu_info()}))
    if not same:
        sys.exit("the routes' files differ")


if __name__ == "__main__":
    main()
