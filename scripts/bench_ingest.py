#!/usr/bin/env python
"""Raw-image ingest on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32): images/s from decoded host uint8 photos of mixed sizes to
detection records, for

  (a) per_image:     Helper.letterbox_device per image into the bound uint8 input, set_image_shapes, step_device and a
                     synchronise per batch (the serving loop before submit_images);
  (b) submit_images: DetectionPipeline.submit_images / collect, two batches in flight.

Both run in one process on one pipeline, after a warm-up of every shape, in alternating windows (three each, median).  The
images are seeded synthetic photos held in host memory, so neither figure includes file decoding; the host-side decode rate of
the same images as PNG and JPEG files is reported separately, per decode thread.  The card's name, power limit and SM clock
are read in the same run.  Prints one JSON line.

    python scripts/bench_ingest.py [--images 256 --batch 32 --windows 3 --passes 8]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from k210_yolo_framework_b200 import Helper  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.yolonet import load_npz_weights  # noqa: E402

SIZES = [(375, 500), (480, 640), (720, 1280), (333, 500), (224, 320)]
GOLDEN = os.path.join(ROOT, "tests", "golden")


def photos(n, seed=0):
    """Smooth colour fields with noise: compress like photos (unlike uniform noise) and span the full 0..255 range."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        f = rng.uniform(0.005, 0.03, 3)
        base = np.stack([127.5 + 127.5 * np.sin(f[c] * (xx + rng.uniform(0, 1) * yy) + rng.uniform(0, 6)) for c in range(3)], -1)
        out.append(np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8))
    return out


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [v.strip() for v in q.split(",")]
    except Exception as e:  # the figures stay unlabelled rather than guessed
        info["nvidia_smi_error"] = repr(e)
    return info


def run_per_image(pipe, helper, buf, batches):
    recs = []
    shapes = np.tile(np.array([pipe.in_hw], np.float32), (pipe.batch, 1))
    for imgs in batches:
        for j, img in enumerate(imgs):
            shapes[j] = img.shape[:2]
            buf[j].copy_(helper.letterbox_device(img))
        pipe.set_image_shapes(shapes)
        pipe.engine.bind_input(buf)
        dets, counts = pipe.step_device(pipe.batch)
        pipe.wait_gathered()
        torch.cuda.synchronize()
        recs.append(DetectionPipeline.records(dets[:len(imgs)].clone(), counts[:len(imgs)].clone()))
    return recs


def run_submit_images(pipe, batches):
    recs, pending = [], []
    for imgs in batches:
        pending.append(pipe.submit_images(imgs))
        if len(pending) == 2:
            recs.append(DetectionPipeline.records(*pipe.collect(pending.pop(0))))
    for t in pending:
        recs.append(DetectionPipeline.records(*pipe.collect(t)))
    return recs


def decode_rate(images, helper, tmp):
    """Images/s of Helper._read_img (PIL) on one thread, per format."""
    from PIL import Image
    out = {}
    for ext, kw in (("png", {}), ("jpg", {"quality": 90})):
        paths = []
        for i, img in enumerate(images):
            p = os.path.join(tmp, f"{i:04d}.{ext}")
            Image.fromarray(img).save(p, **kw)
            paths.append(p)
        helper._read_img(paths[0])
        t0 = time.perf_counter()
        for p in paths:
            helper._read_img(p)
        out[ext] = round(len(paths) / (time.perf_counter() - t0), 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--passes", type=int, default=8, help="passes over the images per window (windows of a second or so)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ingest measures on a GPU"
    torch.cuda.set_device(0)
    H, W = 224, 320
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = DetectionPipeline("yolo_mobilev1", (H, W), anchors, 20, 0.75, args.batch, obj_thresh=0.7, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    helper = Helper(None, 20, anchors, [[H, W]], [[7, 10], [14, 20]])
    buf = torch.zeros((args.batch, H, W, 3), dtype=torch.uint8, device="cuda")
    images = photos(args.images)
    batches = [images[i:i + args.batch] for i in range(0, len(images), args.batch)]

    # warm-up: every shape through both routes (module loads, graph captures, staging growth); both give the same records
    rec_a = run_per_image(pipe, helper, buf, batches)
    rec_b = run_submit_images(pipe, batches)
    same = rec_a == rec_b
    times = {"per_image": [], "submit_images": []}
    for _ in range(args.windows):
        for name, fn in (("per_image", lambda: run_per_image(pipe, helper, buf, batches)),
                         ("submit_images", lambda: run_submit_images(pipe, batches))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = [fn() for _ in range(args.passes)]
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            same = same and all(r == rec_a for r in out)
    gpu = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        dec = decode_rate(images[:2 * len(SIZES) * 4], helper, tmp)
    rate = {k: round(args.passes * len(images) / statistics.median(v), 1) for k, v in times.items()}
    print(json.dumps({
        "metric": "ingest_img_per_s", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}", "images": len(images), "passes": args.passes,
        "sizes": [list(s) for s in SIZES], "per_image": rate["per_image"], "submit_images": rate["submit_images"],
        "speedup": round(rate["submit_images"] / rate["per_image"], 2), "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()},
        "records_equal": same, "host_decode_img_per_s_per_thread": dec, "gpu": gpu}))
    if not same:
        sys.exit("submit_images records differ from the per-image route")


if __name__ == "__main__":
    main()
