#!/usr/bin/env python
"""Video to records on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32): frames/s from a video file to detection records, as
serve.py runs a video (detect_files, two batches in flight), for

  gpu:          Motion-JPEG AVI frames read by index and decoded on the GPU (the route serve.py takes);
  pil_N:        the same frames decoded by PIL in N host threads (1, 4, 16);
  pixels:       the same frames already decoded, in host memory (no decoding at all);
  draw:         the GPU route with --draw: the drawn frames rendered and encoded on the GPU and written as a Motion-JPEG AVI;
  ffmpeg_mp4v:  the same frames as an mp4v video, decoded in order by OpenCV's FFmpeg backend on the host threads.

The video: the bench_ingest photos resized to 1280x720 with the golden dog photo pasted in (so that there are records to
compare), written as a Motion-JPEG AVI at 4:2:2, quality 90, without DHT segments, as cameras write them.  Every route runs
once to warm up and then `--windows` timed passes (median).  All Motion-JPEG routes must give the same records, and the mp4v
route the records of its own decoded pixels; the run fails otherwise.  The card's name, power limit and SM clock are read in
the same run.  Prints one JSON line.

    python scripts/bench_video.py [--frames 256 --batch 32 --windows 3]
"""
import argparse
import io
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import serve  # noqa: E402
from bench_ingest import GOLDEN, gpu_info, photos  # noqa: E402
from k210_yolo_framework_b200.helper import read_image  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.video import AviWriter, jpeg_hw, open_video  # noqa: E402
from k210_yolo_framework_b200.yolonet import load_npz_weights  # noqa: E402

H720, W720 = 720, 1280


def strip_dht(data: bytes) -> bytes:
    """The JPEG file without its DHT segments (the decoder then uses the standard tables, as PIL wrote them)."""
    out, i = bytearray(data[:2]), 2
    while data[i + 1] != 0xDA:
        n = int.from_bytes(data[i + 2:i + 4], "big")
        if data[i + 1] != 0xC4:
            out += data[i:i + 2 + n]
        i += 2 + n
    return bytes(out + data[i:])


def frames_720p(n):
    from PIL import Image
    dog = np.load(os.path.join(GOLDEN, "dog_u8.npy"))
    out = []
    for k, img in enumerate(photos(n)):
        f = np.asarray(Image.fromarray(img).resize((W720, H720), Image.BILINEAR)).copy()
        y, x = (37 * k) % (H720 - dog.shape[0]), (53 * k) % (W720 - dog.shape[1])
        f[y:y + dog.shape[0], x:x + dog.shape[1]] = dog
        out.append(f)
    return out


def run(pipe, n, load, threads, writer_path=None, fps=30.0):
    """Records of frames 0 .. n-1 through detect_files; with `writer_path` the drawn frames go to a Motion-JPEG AVI."""
    recs, writer = [], None
    for item in serve.detect_files(pipe, list(range(n)), threads, load, rendered=writer_path is not None):
        recs += DetectionPipeline.records(item[1], item[2])[:len(item[0])]
        if writer_path is not None:
            for data in item[3]:
                writer = writer or AviWriter(writer_path, fps, jpeg_hw(data))
                writer.write(data)
    if writer is not None:
        writer.close()
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_video measures on a GPU"
    import cv2
    from PIL import Image
    torch.cuda.set_device(0)
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, args.batch, obj_thresh=0.3, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    n = args.frames
    with tempfile.TemporaryDirectory() as tmp:
        avi, mp4 = os.path.join(tmp, "cam.avi"), os.path.join(tmp, "cam.mp4")
        pixels = frames_720p(n)
        w = cv2.VideoWriter(mp4, cv2.CAP_FFMPEG, cv2.VideoWriter_fourcc(*"mp4v"), 30.0, (W720, H720))
        with AviWriter(avi, 30.0, (H720, W720)) as aw:
            for f in pixels:
                b = io.BytesIO()
                Image.fromarray(f).save(b, "JPEG", quality=90, subsampling=1)
                aw.write(strip_dht(b.getvalue()))
                w.write(np.ascontiguousarray(f[..., ::-1]))
        w.release()
        src = open_video(avi)
        avi_bytes, mp4_bytes = os.path.getsize(avi), os.path.getsize(mp4)
        assert src.n_frames == n and src.codec == "MJPG"
        decoded = [read_image(io.BytesIO(src.frame_bytes(k))) for k in range(n)]
        mp4_src = open_video(mp4)
        assert mp4_src.n_frames == n
        mp4_pixels = list(mp4_src.frames())
        gpu_load = src.loader(route=serve.route_image)
        pil_load = src.loader(route=lambda data: read_image(io.BytesIO(data)))
        routes = {
            "gpu": lambda: run(pipe, n, gpu_load, 4),
            "pil_1": lambda: run(pipe, n, pil_load, 1),
            "pil_4": lambda: run(pipe, n, pil_load, 4),
            "pil_16": lambda: run(pipe, n, pil_load, 16),
            "pixels": lambda: run(pipe, n, decoded.__getitem__, 4),
            "ffmpeg_mp4v": lambda: run(pipe, n, mp4_src.loader(), 4),
        }
        gpu_frames = sum(serve.gpu_decodable(src.frame_bytes(k)) for k in range(n))
        recs = {name: fn() for name, fn in routes.items()}       # warm-up of every route
        mp4_ref = run(pipe, n, mp4_pixels.__getitem__, 4)
        times = {name: [] for name in routes}
        for _ in range(args.windows):
            for name, fn in routes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
                recs[name] = recs[name] if out == recs[name] else None
        pipe.enable_rendering(quality=75)
        drawn = os.path.join(tmp, "drawn.avi")
        recs["draw"] = run(pipe, n, gpu_load, 4, drawn)
        times["draw"] = []
        for _ in range(args.windows):
            t0 = time.perf_counter()
            out = run(pipe, n, gpu_load, 4, drawn)
            times["draw"].append(time.perf_counter() - t0)
            recs["draw"] = recs["draw"] if out == recs["draw"] else None
        drawn_frames = open_video(drawn).n_frames
        gpu = gpu_info()
    mjpeg = [recs[k] for k in ("gpu", "pil_1", "pil_4", "pil_16", "pixels", "draw")]
    same = all(r is not None and r == mjpeg[0] for r in mjpeg) and recs["ffmpeg_mp4v"] == mp4_ref and drawn_frames == n
    rate = {k: round(n / statistics.median(v), 1) for k, v in times.items()}
    print(json.dumps({
        "metric": "video_frames_per_s", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}", "frames": n,
        "video": f"MJPEG AVI {W720}x{H720} 4:2:2 q90 without DHT", "avi_bytes": avi_bytes, "mp4v_bytes": mp4_bytes,
        "gpu_decoded_frames": int(gpu_frames), "records": int(sum(len(r) for r in mjpeg[0] or [])), "frames_per_s": rate,
        "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()}, "records_equal": same, "gpu": gpu}))
    if not same:
        sys.exit("the routes' records differ")


if __name__ == "__main__":
    main()
