#!/usr/bin/env python
"""GPU PNG decode on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32), one process, one GPU.  The images are bench_ingest's
seeded photos (five sizes, 375x500 to 720x1280) encoded once as PNG files in memory, by PIL (default level) and by cv2 (its
defaults; `--encoder`).  Reports:

  decode:        the decode kernels (k2y_png_decode) per batch of 32, timed with CUDA events over many batches, as images/s,
                 compressed and inflated MB/s, chunks per image, the share of speculative chunks confirmed on the chain, the
                 bytes per image the longest single decoder inflated (the serial part), and each kernel's share from
                 torch.profiler (device time per batch, by kernel);
  records/s:     file bytes -> detection records through DetectionPipeline.submit_images(bytes) with enable_png_decode
                 (two batches in flight),
                 against submit_images of the same files decoded by PIL (Helper._read_img) in 1, 4 and 16 host threads,
                 one batch ahead as serve.py does, and against submit_images of the already decoded pixels (the pipeline
                 without any file decode); alternating windows, median of three;
  records_equal: every route gives the same records (the run fails otherwise);

and the card's name, power limit and SM clock, read in the same run.  Prints one JSON line.

    python scripts/bench_png.py [--encoder pil|cv2 --images 256 --batch 32 --windows 3 --passes 4 --decode_reps 20]
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


def png_files(images, encoder):
    if encoder == "cv2":
        import cv2
        return [cv2.imencode(".png", np.ascontiguousarray(img[..., ::-1]))[1].tobytes() for img in images]
    from PIL import Image
    out = []
    for img in images:
        b = io.BytesIO()
        Image.fromarray(img).save(b, "PNG")
        out.append(b.getvalue())
    return out


def time_decode(files, reps):
    """Device ms per k2y_png_decode of `files` (events around `reps` back-to-back calls) and the status words."""
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    layout = preprocess.BatchLayout(files, (224, 320), gpu_png=True)
    dst_offsets = layout.offsets.astype(np.int64)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev)
    staging = preprocess.Staging(dev, st)
    staging.reserve(layout.png_plan[3], len(files))
    preprocess.stage_pngs(bufs, dst_offsets, staging, layout.png_plan, staging.dev)
    _, blob_at, blob_bytes, _ = layout.png_plan
    blob = staging.host.numpy()[blob_at:blob_at + blob_bytes]

    def once():
        check(lib.k2y_png_decode(blob.ctypes.data, staging.dev.data_ptr() + blob_at, staging.dev.data_ptr(), staging.dev.data_ptr(),
                                 staging.png_workspace.data_ptr(), staging.png_workspace.numel(), staging.png_status.data_ptr(),
                                 ctypes.c_void_p(st.cuda_stream)))
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
    for e in prof.key_averages():
        for k in ("png_gather_kernel", "png_find_kernel", "png_chunk_kernel", "png_resolve_kernel", "png_inflate_kernel",
                  "png_unfilter_kernel"):
            if k in e.key:
                kernels[k] = kernels.get(k, 0.0) + e.device_time_total / 1e3 / prof_reps
        if "emset" in e.key:
            kernels["memset"] = kernels.get("memset", 0.0) + e.device_time_total / 1e3 / prof_reps
    return ms, kernels, staging.png_status[:len(files)].cpu().numpy()


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
    ap.add_argument("--decode_reps", type=int, default=20, help="decode calls timed per batch")
    ap.add_argument("--encoder", choices=["pil", "cv2"], default="pil")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_png measures on a GPU"
    torch.cuda.set_device(0)
    files = png_files(photos(args.images), args.encoder)
    assert all(preprocess.png_gpu_decodable(f) for f in files)
    batches = [files[i:i + args.batch] for i in range(0, len(files), args.batch)]

    # (1) the decode kernels alone, per batch of `batch` files
    ms, chunks, confirmed, serial, kernel_ms = [], 0, 0, 0, {}
    for b in batches:
        t, kern, status = time_decode(b, args.decode_reps)
        assert (status[:, 0] == 0).all(), status
        ms.append(t)
        for k, v in kern.items():
            kernel_ms[k] = kernel_ms.get(k, 0.0) + v / len(batches)
        chunks += int(status[:, 1].sum())
        confirmed += int(status[:, 2].sum())
        serial += int(status[:, 3].sum())
    per_batch = statistics.mean(ms)
    mb = sum(len(f) for f in files) / len(batches) / 1e6
    inflated = sum(preprocess.inspect_png(f)[0] * (1 + preprocess.inspect_png(f)[1] * 3) for f in files)

    # (2) records/s from file bytes
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, args.batch, obj_thresh=0.7, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    pipe.enable_png_decode()
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
        "metric": "png_decode", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}", "images": len(files),
        "sizes": [list(s) for s in SIZES], "png": {"pil": "PIL, default level", "cv2": "cv2.imencode defaults"}[args.encoder],
        "compressed_mb_per_batch": round(mb, 3), "inflated_mb_per_batch": round(inflated / len(batches) / 1e6, 3),
        "decode_ms_per_batch": round(per_batch, 4), "decode_img_per_s": round(args.batch / per_batch * 1e3, 1),
        "decode_compressed_mb_per_s": round(mb / per_batch * 1e3, 1),
        "decode_inflated_mb_per_s": round(inflated / len(batches) / 1e6 / per_batch * 1e3, 1),
        "chunks_per_image": round(chunks / len(files), 2),
        "confirmed_chunk_rate": round(confirmed / max(1, chunks - len(files)), 4),
        "serial_bytes_per_image": round(serial / len(files)),
        "decode_kernel_ms_per_batch": {k: round(v, 4) for k, v in kernel_ms.items()},
        "records_per_s": rate,
        "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()}, "records_equal": same, "gpu": gpu_info()}))
    if not same:
        sys.exit("the routes' records differ")


if __name__ == "__main__":
    main()
