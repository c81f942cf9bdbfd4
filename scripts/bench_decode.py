#!/usr/bin/env python
"""GPU JPEG decode on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32), one process, one GPU.  The images are bench_ingest's
seeded photos (five sizes, 375x500 to 720x1280) encoded once as JPEG files in memory (PIL, quality 90, 4:2:0).  Reports:

  decode:        the five decode kernels (k2y_jpeg_decode) per batch of 32, timed with CUDA events over many batches, as
                 images/s and compressed MB/s, with the mean and maximum synchronisation rounds per window of subsequences,
                 and each kernel's share from torch.profiler (device time per batch, by kernel);
  records/s:     file bytes -> detection records through DetectionPipeline.submit_images(bytes) (two batches in flight),
                 against submit_images of the same files decoded by PIL (Helper._read_img) in 1, 4 and 16 host threads,
                 one batch ahead as serve.py does, and against submit_images of the already decoded pixels (the pipeline
                 without any file decode); alternating windows, median of three;
  records_equal: every route gives the same records (the run fails otherwise);

and the card's name, power limit and SM clock, read in the same run.  Prints one JSON line.

With --progressive the files are the same photos saved by PIL as progressive JPEGs (quality 90, 4:2:0, libjpeg's default
scan script), the decode is k2y_jpeg_progressive_decode (the pipeline's enable_progressive_jpeg_decode), the kernel split
gives each entropy-decode level on its own (level 0: the DC, chroma and luma 1..5 first scans; level 1: the luma 6..63
first scan and the DC and chroma refinements; levels 2 and 3: the luma refinements), and the JSON adds
the host milliseconds BatchLayout takes to parse and plan a batch of the files and to write its descriptor blob.

    python scripts/bench_decode.py [--progressive] [--images 256 --batch 32 --windows 3 --passes 4 --decode_reps 50]
"""
import argparse
import ctypes
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
from bench_ingest import GOLDEN, SIZES, gpu_info, photos  # noqa: E402
from k210_yolo_framework_b200 import preprocess  # noqa: E402
from k210_yolo_framework_b200._lib import check, lib  # noqa: E402
from k210_yolo_framework_b200.helper import read_image  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.yolonet import load_npz_weights  # noqa: E402


def jpeg_files(images, progressive=False):
    from PIL import Image
    out = []
    for img in images:
        b = io.BytesIO()
        Image.fromarray(img).save(b, "JPEG", quality=90, progressive=progressive)
        out.append(b.getvalue())
    return out


def time_decode(files, reps, progressive=False):
    """Device ms per k2y_jpeg_decode (k2y_jpeg_progressive_decode) of `files` (events around `reps` back-to-back calls),
    the per-kernel split and the status words."""
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    layout = preprocess.BatchLayout(files, (224, 320), gpu_progressive=progressive)
    dst_offsets = layout.offsets.astype(np.int64)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev)
    staging = preprocess.Staging(dev, st)
    plan = layout.progressive_plan if progressive else layout.jpeg_plan
    staging.reserve(plan[3], len(files))
    (preprocess.stage_progressive_jpegs if progressive else preprocess.stage_jpegs)(bufs, dst_offsets, staging, plan, staging.dev)
    _, blob_at, blob_bytes, _ = plan
    blob = staging.host.numpy()[blob_at:blob_at + blob_bytes]
    decode = lib.k2y_jpeg_progressive_decode if progressive else lib.k2y_jpeg_decode
    ws = staging.progressive_workspace if progressive else staging.workspace
    status = staging.progressive_status if progressive else staging.status

    def once():
        check(decode(blob.ctypes.data, staging.dev.data_ptr() + blob_at, staging.dev.data_ptr(), staging.dev.data_ptr(),
                     ws.data_ptr(), ws.numel(), status.data_ptr(), ctypes.c_void_p(st.cuda_stream)))
    for _ in range(3):
        once()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(st)
    for _ in range(reps):
        once()
    t1.record(st)
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    # per-kernel device time of the same calls
    from torch.profiler import ProfilerActivity, profile
    prof_reps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(prof_reps):
            once()
        torch.cuda.synchronize()
    kernels = {}
    names = ("prog_idct_kernel", "prog_color_kernel") if progressive else \
        ("jpeg_unstuff_kernel", "jpeg_huffman_kernel", "jpeg_dc_kernel", "jpeg_idct_kernel", "jpeg_color_kernel")
    for e in prof.key_averages():
        for k in names:
            if k in e.key:
                kernels[k] = kernels.get(k, 0.0) + e.device_time_total / 1e3 / prof_reps
        if "emset" in e.key:
            kernels["memset"] = kernels.get("memset", 0.0) + e.device_time_total / 1e3 / prof_reps
    if progressive:     # the entropy launches of one call, in launch order: one per level
        launches = sorted((e.time_range.start, e.time_range.elapsed_us()) for e in prof.events()
                          if "prog_entropy_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA)
        levels = len(launches) // prof_reps
        for i, (_, us) in enumerate(launches):
            k = f"prog_entropy_kernel_level_{i % levels}"
            kernels[k] = kernels.get(k, 0.0) + us / 1e3 / prof_reps
    return ms, kernels, status[:len(files)].cpu().numpy()


def run_bytes(pipe, batches):
    recs, pending = [], []
    for files in batches:
        pending.append(pipe.submit_images(files))
        if len(pending) == 2:
            recs.append(DetectionPipeline.records(*pipe.collect(pending.pop(0))))
    for t in pending:
        recs.append(DetectionPipeline.records(*pipe.collect(t)))
    return recs


def run_pil(pipe, batches, pool):
    recs, pending = [], []
    nxt = [pool.submit(read_image, io.BytesIO(f)) for f in batches[0]]
    for g in range(len(batches)):
        imgs = [f.result() for f in nxt]
        nxt = [pool.submit(read_image, io.BytesIO(f)) for f in batches[g + 1]] if g + 1 < len(batches) else []
        pending.append(pipe.submit_images(imgs))
        if len(pending) == 2:
            recs.append(DetectionPipeline.records(*pipe.collect(pending.pop(0))))
    for t in pending:
        recs.append(DetectionPipeline.records(*pipe.collect(t)))
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--passes", type=int, default=4, help="passes over the images per window")
    ap.add_argument("--decode_reps", type=int, default=50, help="decode calls timed per batch")
    ap.add_argument("--progressive", action="store_true", help="progressive JPEG files and the progressive decoder")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_decode measures on a GPU"
    torch.cuda.set_device(0)
    files = jpeg_files(photos(args.images), args.progressive)
    assert all((preprocess.progressive_gpu_decodable if args.progressive else preprocess.gpu_decodable)(f) for f in files)
    batches = [files[i:i + args.batch] for i in range(0, len(files), args.batch)]

    # (0) host: BatchLayout's parse and plan of a batch, and the blob it writes
    host_layout_ms, host_blob_ms = [], []
    for b in batches:
        t0 = time.perf_counter()
        lay = preprocess.BatchLayout(b, (224, 320), gpu_progressive=args.progressive)
        t1 = time.perf_counter()
        plan = lay.progressive_plan if args.progressive else lay.jpeg_plan
        blob = np.zeros(plan[2] + 16, np.uint8)
        blob = blob[(-blob.ctypes.data) % 16:][:plan[2]]
        t2 = time.perf_counter()
        (preprocess._progressive_plan if args.progressive else preprocess._jpeg_plan)(
            [np.frombuffer(f, np.uint8) for f in b], plan[0], lay.offsets.astype(np.int64), blob)
        t3 = time.perf_counter()
        host_layout_ms.append((t1 - t0) * 1e3)
        host_blob_ms.append((t3 - t2) * 1e3)

    # (1) the decode kernels alone, per batch of `batch` files
    ms, rounds_max, rounds_sum, windows, kernel_ms = [], 0, 0, 0, {}
    for b in batches:
        t, kern, status = time_decode(b, args.decode_reps, args.progressive)
        assert (status[:, 0] == 0).all(), status
        ms.append(t)
        for k, v in kern.items():
            kernel_ms[k] = kernel_ms.get(k, 0.0) + v / len(batches)
        rounds_max = max(rounds_max, int(status[:, 1].max()))   # (zero for progressive files: no speculation)
        rounds_sum += int(status[:, 2].sum())
        windows += int(status[:, 3].sum())
    per_batch = statistics.mean(ms)
    mb = sum(len(f) for f in files) / len(batches) / 1e6

    # (2) records/s from file bytes
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, args.batch, obj_thresh=0.7, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    if args.progressive:
        pipe.enable_progressive_jpeg_decode()
    threads = (1, 4, 16)
    pools = {k: ThreadPoolExecutor(k) for k in threads}
    pixels = [[read_image(io.BytesIO(f)) for f in b] for b in batches]
    routes = {"gpu_decode": lambda: run_bytes(pipe, batches), "decoded_pixels": lambda: run_bytes(pipe, pixels)}
    for k in threads:
        routes[f"pil_{k}_threads"] = (lambda k=k: run_pil(pipe, batches, pools[k]))
    ref = routes["gpu_decode"]()
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
        "metric": "jpeg_progressive_decode" if args.progressive else "jpeg_decode",
        "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}", "images": len(files),
        "sizes": [list(s) for s in SIZES], "jpeg": "PIL quality 90, 4:2:0" + (", progressive" if args.progressive else ""),
        "compressed_mb_per_batch": round(mb, 3),
        "host_layout_ms_per_batch": round(statistics.median(host_layout_ms), 3),
        "host_blob_ms_per_batch": round(statistics.median(host_blob_ms), 3),
        "decode_ms_per_batch": round(per_batch, 4), "decode_img_per_s": round(args.batch / per_batch * 1e3, 1),
        "decode_mb_per_s": round(mb / per_batch * 1e3, 1), "sync_rounds_mean": round(rounds_sum / max(windows, 1), 3),
        "sync_rounds_max": rounds_max, "decode_kernel_ms_per_batch": {k: round(v, 4) for k, v in kernel_ms.items()},
        "records_per_s": rate,
        "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()}, "records_equal": same, "gpu": gpu_info()}))
    if not same:
        sys.exit("the routes' records differ")


if __name__ == "__main__":
    main()
