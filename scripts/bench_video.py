#!/usr/bin/env python
"""Video to records on cfg 2 (yolo_mobilev1 0.75, 224x320, batch 32): frames/s from a video file to detection records, as
serve.py runs a video (detect_files, two batches in flight), for

  gpu:          Motion-JPEG AVI frames read by index and decoded on the GPU (the route serve.py takes);
  pil_N:        the same frames decoded by PIL in N host threads (1, 4, 16);
  pixels:       the same frames already decoded, in host memory (no decoding at all);
  draw:         the GPU route with --draw: the drawn frames rendered and encoded on the GPU and written as a Motion-JPEG AVI;
  ffmpeg_mp4v:  the same frames as an mp4v video, decoded in order by OpenCV's FFmpeg backend on the host threads.

With --track, also SORT tracking of the same records (DetectionPipeline.enable_tracking, default setting):
  gpu_plain /    the GPU route on two fresh pipelines, one tracking on the GPU (one k2y_track_update launch per batch, behind
  gpu_track:     the NMS) and one not, their windows alternating (which goes first alternates too);
  track_kernel:  that kernel's time per batch of frames, from CUDA events around its launches, on the route's records and on
                 two dense synthetic streams: "dense_voc" (20 classes, each with about 27 of its 30 records in every frame,
                 moving objects) and "coco_bound" (80 classes of 100, max_age 9, one class with 100 new records in every frame,
                 so that it holds its bound of 1000 tracks);
  sort_ref /     the route's records and the dense_voc stream tracked on the host by oracle/sort_ref.py (scalar filter,
  sort_matrix:   plain-Python assignment) and by a literal matrix-form SORT (numpy filter, iou_batch, scipy's
                 linear_sum_assignment), frames/s of the tracker alone: scipy imported and one pass run before the timed
                 windows (median).
The GPU's ids and boxes must equal sort_ref's; the run fails otherwise.

With --track bytetrack, also ByteTrack (DetectionPipeline.enable_tracking(method="bytetrack"), default setting) beside the SORT
arms, on pipelines at obj_thresh 0.1 so that the low-score association has records:
  gpu_plain /    the GPU route on two fresh pipelines, one tracking with k2y_bytetrack_update and one not, windows alternating;
  gpu_track:
  bytetrack_kernel:  the kernel's time per batch of frames, from CUDA events around its launches, on the route's records, on
                 the "dense_voc" stream of the SORT arms with scores (0.9, or 0.3 for a record with probability 0.15) and at
                 "coco_bound" (80 classes of 100, track_buffer 30, class 0 given 100 new boxes every second frame, which it
                 confirms the frame after and then loses, so that its lost tracks pile up to about 1,600);
  bytetrack_ref: the route's records and the first batch of dense_voc tracked on the host by oracle/bytetrack_ref.py,
                 frames/s of the tracker alone (one pass run first, median).
The GPU's ids and boxes on the route's records and on the first batch of dense_voc must equal bytetrack_ref's; the run fails
otherwise.

With --track ocsort, the same arms for OC-SORT (DetectionPipeline.enable_tracking(method="ocsort"), default setting) on
pipelines at the default obj_thresh 0.3: gpu_plain / gpu_track, ocsort_kernel (k2y_ocsort_update on the route's records, on the
scored dense_voc stream and at "coco_bound", 80 classes of 100 with max_age 39, class 0 given 100 new boxes in every frame so
that it holds its bound of 4,000 tracks) and ocsort_ref (oracle/ocsort_ref.py on the host).  The GPU's ids and boxes on the
route's records and on the first batch of dense_voc must equal ocsort_ref's; the run fails otherwise.

With --draw_tracks, also the track drawing (DetectionPipeline.enable_rendering(tracks=True), SORT, default setting):
  draw_plain /   the GPU route with --track --draw on two fresh pipelines, one drawing the records and one the tracks
  draw_tracks:   (--draw_tracks), windows alternating; every frame of the tracks' AVI must equal draw.draw_tracks of the
                 frame with its tracks + PIL's save, byte for byte, and the records of both must equal the gpu route's;
  render_kernel: CUDA-event time of k2y_render_tracks and of k2y_render_detections on the same 32 decoded frames, drawing
                 that batch's tracks and records: windows of 50 launches enqueued back to back on one stream through the
                 packed entry points (colour tables and atlases built once, no synchronise between launches), the two
                 kernels' windows alternating, median of the windows.

The video: the bench_ingest photos resized to 1280x720 with the golden dog photo pasted in (so that there are records to
compare), written as a Motion-JPEG AVI at 4:2:2, quality 90, without DHT segments, as cameras write them.  Every route runs
once to warm up and then `--windows` timed passes (median).  All Motion-JPEG routes must give the same records, and the mp4v
route the records of its own decoded pixels; the run fails otherwise.  The card's name, power limit and SM clock are read in
the same run.  Prints one JSON line.

    python scripts/bench_video.py [--frames 256 --batch 32 --windows 3 --track [bytetrack | ocsort] --draw_tracks]
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


def run(pipe, n, load, threads, writer_path=None, fps=30.0, tracks=None):
    """Records of frames 0 .. n-1 through detect_files; with `writer_path` the drawn frames go to a Motion-JPEG AVI; with
    `tracks` (a list; the pipeline's tracking enabled) the frames are tracked and each batch's (ids, boxes) copies go there."""
    recs, writer = [], None
    positions = list(range(n)) if tracks is not None else None
    for item in serve.detect_files(pipe, list(range(n)), threads, load, rendered=writer_path is not None, positions=positions):
        recs += DetectionPipeline.records(item[1], item[2])[:len(item[0])]
        if tracks is not None:
            tracks.append((item[-1][0].clone(), item[-1][1].clone()))
        if writer_path is not None:
            for data in item[3]:
                writer = writer or AviWriter(writer_path, fps, jpeg_hw(data))
                writer.write(data)
    if writer is not None:
        writer.close()
    return recs


def new_pipeline(anchors, batch, obj_thresh=0.3):
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), anchors, 20, 0.75, batch, obj_thresh=obj_thresh, iou_thresh=0.5)
    pipe.engine.set_weights(load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    return pipe


SCORED = {"bytetrack": "ByteTrack", "ocsort": "OC-SORT"}     # the --track arms beside SORT's


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--track", nargs="?", const="sort", default=None, choices=["sort", "bytetrack", "ocsort"],
                    help="also measure SORT tracking on the GPU and on the host; `--track bytetrack` measures ByteTrack too, "
                         "`--track ocsort` OC-SORT")
    ap.add_argument("--draw_tracks", action="store_true", help="also measure drawing the tracks (route and kernel)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_video measures on a GPU"
    import cv2
    from PIL import Image
    torch.cuda.set_device(0)
    anchors = np.load(os.path.join(GOLDEN, "voc_anchor.npy"))
    pipe = new_pipeline(anchors, args.batch)
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
        make_pipe = lambda obj_thresh=0.3: new_pipeline(anchors, args.batch, obj_thresh)     # noqa: E731
        track = bench_track(make_pipe, n, gpu_load, recs["gpu"], args.batch, args.windows) if args.track else None
        scored = bench_scored(make_pipe, n, gpu_load, args.batch, args.windows, args.track) if args.track in SCORED else None
        drawing = bench_draw_tracks(make_pipe, n, src, gpu_load, decoded, recs["gpu"], args.batch, args.windows, tmp) \
            if args.draw_tracks else None
        gpu = gpu_info()
    mjpeg = [recs[k] for k in ("gpu", "pil_1", "pil_4", "pil_16", "pixels", "draw")]
    same = all(r is not None and r == mjpeg[0] for r in mjpeg) and recs["ffmpeg_mp4v"] == mp4_ref and drawn_frames == n
    rate = {k: round(n / statistics.median(v), 1) for k, v in times.items()}
    print(json.dumps({
        "metric": "video_frames_per_s", "cfg": f"yolo_mobilev1 alpha 0.75, 224x320, batch {args.batch}", "frames": n,
        "video": f"MJPEG AVI {W720}x{H720} 4:2:2 q90 without DHT", "avi_bytes": avi_bytes, "mp4v_bytes": mp4_bytes,
        "gpu_decoded_frames": int(gpu_frames), "records": int(sum(len(r) for r in mjpeg[0] or [])), "frames_per_s": rate,
        "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()}, "records_equal": same,
        **({"track": track} if track else {}), **({args.track: scored} if scored else {}),
        **({"draw_tracks": drawing} if drawing else {}), "gpu": gpu}))
    if not same:
        sys.exit("the routes' records differ")
    if track and not track["ids_equal"]:
        sys.exit("the GPU tracker's ids and boxes differ from oracle/sort_ref.py's")
    if scored and not scored["ids_equal"]:
        sys.exit(f"the GPU {SCORED[args.track]}'s ids and boxes differ from oracle/{args.track}_ref.py's")
    if drawing and not (drawing["frames_equal_pil"] and drawing["records_equal"]):
        sys.exit("the drawn tracks differ from draw.draw_tracks + PIL's save, or the records from the gpu route's")


def draw_tracks_of(img, k, tracks, recs, batch, colormap):
    """Frame k drawn by draw.draw_tracks with its tracks (the route's per-batch (ids, boxes) and per-frame records), saved as
    PIL saves it at quality 75."""
    from k210_yolo_framework_b200.draw import draw_tracks
    ids, boxes = (x[k % batch].numpy() for x in tracks[k // batch])
    seen, found = {}, []
    for c, *_ in recs[k]:
        j = seen[c] = seen.get(c, -1) + 1
        found.append((c, int(ids[c, j]), *(float(v) for v in boxes[c, j])))
    b = io.BytesIO()
    draw_tracks(img, found, colormap).save(b, "JPEG", quality=75)
    return b.getvalue()


def bench_draw_tracks(make_pipe, n, src, load, decoded, gpu_recs, batch, windows, tmp):
    """The --draw_tracks arms: --track --draw against --track --draw --draw_tracks on the route, and k2y_render_tracks
    against k2y_render_detections on one batch of decoded frames."""
    from k210_yolo_framework_b200.helper import _COLORMAP
    from k210_yolo_framework_b200.render import (LabelAtlas, TrackLabelAtlas, color_table, render_packed, render_tracks_packed,
                                                 track_color_table)
    pipes, paths, tracks, recs = {}, {}, {}, {}
    for name, on in (("draw_plain", False), ("draw_tracks", True)):
        pipes[name] = make_pipe()
        pipes[name].enable_tracking()
        pipes[name].enable_rendering(quality=75, tracks=on)
        paths[name] = os.path.join(tmp, f"{name}.avi")
    times = {name: [] for name in pipes}
    for w in range(windows + 1):          # window 0 warms up; the order alternates
        for name in (list(pipes) if w % 2 == 0 else list(pipes)[::-1]):
            pipes[name].reset_tracks()
            tracks[name] = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            recs[name] = run(pipes[name], n, load, 4, paths[name], tracks=tracks[name])
            torch.cuda.synchronize()
            if w:
                times[name].append(time.perf_counter() - t0)
    drawn = open_video(paths["draw_tracks"])
    frames_equal = drawn.n_frames == n and all(
        drawn.frame_bytes(k) == draw_tracks_of(decoded[k], k, tracks["draw_tracks"], recs["draw_tracks"], batch, _COLORMAP)
        for k in range(n))
    # the kernels: the first batch's frames, records and tracks on the device
    m = min(batch, n)
    pipe = make_pipe()
    pipe.enable_tracking()
    t = pipe.submit_images([src.frame_bytes(k) for k in range(m)], frames=list(range(m)))
    dets, counts = (x[:m].cuda() for x in pipe.collect(t))
    ids, boxes = (x[:m].cuda() for x in pipe.tracks(t))
    buf = torch.empty((m, H720, W720, 3), dtype=torch.uint8, device="cuda")
    buf.copy_(torch.from_numpy(np.stack(decoded[:m])))
    # the packed entry points with colour tables built once and atlases uploaded by the warm-up: nothing but the launch's host
    # setup between two launches, no synchronise
    dev, st = buf.device, torch.cuda.current_stream()
    offsets = np.arange(m, dtype=np.int64) * (H720 * W720 * 3)
    hw = np.array([[H720, W720]] * m, np.int32)
    det_atlas, track_atlas = LabelAtlas(20), TrackLabelAtlas()
    det_colors, track_colors = color_table(_COLORMAP, 20, dev), track_color_table(_COLORMAP, dev)
    calls = {"render_detections": lambda: render_packed(buf.data_ptr(), offsets, hw, dets, counts, det_atlas, det_colors, dev, st),
             "render_tracks": lambda: render_tracks_packed(buf.data_ptr(), offsets, hw, counts, ids, boxes, track_atlas,
                                                           track_colors, dev, st)}
    for fn in calls.values():
        fn()
    kernel = {name: [] for name in calls}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for w in range(max(windows, 5)):
        for name in (list(calls) if w % 2 == 0 else list(calls)[::-1]):
            ev[0].record()
            for _ in range(50):
                calls[name]()
            ev[1].record()
            ev[1].synchronize()
            kernel[name].append(ev[0].elapsed_time(ev[1]) / 50)
    return {"frames_per_s": {k: round(n / statistics.median(v), 1) for k, v in times.items()},
            "windows_s": {k: [round(x, 4) for x in v] for k, v in times.items()},
            "render_kernel_ms_per_batch": {k: round(statistics.median(v), 4) for k, v in kernel.items()},
            "kernel_batch": f"{m} frames {W720}x{H720}, {int(counts.clamp(min=0).sum())} records, "
                            f"{int((ids >= 0).sum())} with a track",
            "tracks_drawn": int(sum(int((i >= 0).sum()) for i, _ in tracks["draw_tracks"])),
            "records_equal": recs["draw_plain"] == gpu_recs and recs["draw_tracks"] == gpu_recs,
            "frames_equal_pil": bool(frames_equal)}


def frame_blocks(recs, C, K, scores=False):
    """Each frame's records as (boxes float32 [C, K, 4], counts [C]), in record order per class; with `scores` also their
    scores float32 [C, K]."""
    out = []
    for frame in recs:
        boxes, counts, sc = np.zeros((C, K, 4), np.float32), np.zeros(C, np.int32), np.zeros((C, K), np.float32)
        for c, _, s, t, l, b, r in frame:
            boxes[c, counts[c]] = (t, l, b, r)
            sc[c, counts[c]] = s
            counts[c] += 1
        out.append((boxes, counts, sc) if scores else (boxes, counts))
    return out


def with_scores(blocks, seed=1):
    """The blocks with a score for each record: 0.9, or 0.3 (an occluded object, ByteTrack's low band) with probability 0.15."""
    rng = np.random.default_rng(seed)
    return [(b, c, np.where(rng.random(b.shape[:2]) < 0.15, 0.3, 0.9).astype(np.float32)) for b, c in blocks]


def bytetrack_bound_blocks(C, K, n):
    """Class 0 piles up lost tracks: K new 10 x 10 high-score boxes every second frame, repeated in the frame after (which
    confirms them) and then left, so that each pair of frames adds K lost tracks until track_buffer removes them."""
    out = []
    for f in range(n):
        boxes, counts, sc = np.zeros((C, K, 4), np.float32), np.zeros(C, np.int32), np.zeros((C, K), np.float32)
        for i in range(K):
            y, x = 40.0 * i, 100.0 + 40.0 * (f // 2)
            boxes[0, i] = (y, x, y + 10, x + 10)
        counts[0] = K
        sc[0, :K] = 0.9
        out.append((boxes, counts, sc))
    return out


def dense_voc_blocks(C, K, n, seed=0):
    """Every class full: K objects of 40 x 40 px on a 60 px lattice (none overlaps another) moving 2 px per frame with noise,
    each record left out of a frame with probability 0.1."""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(n):
        boxes, counts = np.zeros((C, K, 4), np.float32), np.zeros(C, np.int32)
        for c in range(C):
            keep = [i for i in range(K) if rng.random() >= 0.1]
            for k, i in enumerate(keep):
                y, x = 60.0 * i + rng.normal(), 60.0 * c + 2.0 * f + rng.normal()
                boxes[c, k] = (y, x, y + 40, x + 40)
            counts[c] = len(keep)
        out.append((boxes, counts))
    return out


def bound_blocks(C, K, n):
    """Class 0 holds its track bound: K new 10 x 10 boxes in every frame that overlap nothing, so every record is born."""
    out = []
    for f in range(n):
        boxes, counts = np.zeros((C, K, 4), np.float32), np.zeros(C, np.int32)
        for i in range(K):
            y, x = 20.0 * i, 100.0 + 20.0 * f
            boxes[0, i] = (y, x, y + 10, x + 10)
        counts[0] = K
        out.append((boxes, counts))
    return out


def time_kernel(blocks, C, K, max_age, batch, windows, dev, make_tracker=None, first=None):
    """(median, max) ms per launch of k2y_track_update (or of the tracker `make_tracker` makes) over the frames in batches
    of `batch`, from CUDA events; the frames' records (and scores, with a third item) staged on the device as gather blocks
    first, one untimed pass to warm up.  With `first` (a list) the first batch's (ids, boxes) of the last pass go there."""
    from k210_yolo_framework_b200.dist import DetectionGather
    from k210_yolo_framework_b200.track import Tracker
    staged = []
    for a in range(0, len(blocks), batch):
        buf = torch.zeros((batch, C * (K * 6 + 1)), dtype=torch.int32)
        d, c = DetectionGather.split(buf, C, K)
        for i, blk in enumerate(blocks[a:a + batch]):
            d[i, :, :, :4] = torch.from_numpy(blk[0].view(np.int32))
            if len(blk) > 2:
                d[i, :, :, 4] = torch.from_numpy(blk[2].view(np.int32))
            c[i] = torch.from_numpy(blk[1])
        m = len(blocks[a:a + batch])
        staged.append((DetectionGather.split(buf.to(dev), C, K), m, torch.arange(a, a + m, dtype=torch.int64, device=dev), a + m - 1))
    rows = torch.arange(batch, dtype=torch.int32, device=dev)
    ids_d = torch.empty((batch, C, K), dtype=torch.int32, device=dev)
    boxes_d = torch.empty((batch, C, K, 4), dtype=torch.float32, device=dev)
    tracker = make_tracker() if make_tracker else Tracker(C, K, max_age=max_age, device=dev.index)
    st = torch.cuda.current_stream()
    per_batch = []
    for w in range(windows + 1):
        tracker.reset()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(staged))]
        for i, ((d, c), m, pos, last) in enumerate(staged):
            ev[2 * i].record(st)
            tracker.update(d, c, rows, pos, m, ids_d, boxes_d, st, last)
            ev[2 * i + 1].record(st)
            if i == 0 and w == windows and first is not None:
                first += [ids_d[:m].cpu().numpy(), boxes_d[:m].cpu().numpy()]
        torch.cuda.synchronize()
        if w:
            per_batch += [ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(len(staged))]
    return round(statistics.median(per_batch), 4), round(max(per_batch), 4)


def bench_track(make_pipe, n, load, recs, batch, windows):
    """The --track arms (see the module docstring)."""
    import scipy.optimize  # noqa: F401  (imported before the host trackers' timing)
    from oracle import sort_ref
    plain, tracked = make_pipe(), make_pipe()
    C, K = plain.gather.C, plain.gather.K
    blocks = frame_blocks(recs, C, K)
    tracked.enable_tracking()
    got = []
    assert run(plain, n, load, 4) == recs                           # warm-up of both
    assert run(tracked, n, load, 4, tracks=got) == recs             # tracking leaves the records as they were
    times = {"gpu_plain": [], "gpu_track": []}
    for w in range(windows):
        arms = ["gpu_plain", "gpu_track"] if w % 2 == 0 else ["gpu_track", "gpu_plain"]
        for arm in arms:
            if arm == "gpu_track":
                tracked.reset_tracks()
                got = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run(tracked, n, load, 4, tracks=got) if arm == "gpu_track" else run(plain, n, load, 4)
            torch.cuda.synchronize()
            times[arm].append(time.perf_counter() - t0)
            assert out == recs
    ids = torch.cat([g[0] for g in got]).numpy()
    boxes = torch.cat([g[1] for g in got]).numpy()
    dense = dense_voc_blocks(C, K, n)
    host = {}
    for stream, frames in (("route", blocks), ("dense_voc", dense)):
        for name, cls in (("sort_ref", sort_ref.Sort), ("sort_matrix", sort_ref.MatrixSort)):
            key = f"{name}_{stream}"
            host[key] = []
            for w in range(windows + 1):        # the first pass warms up
                tracker = cls(C, K)
                t0 = time.perf_counter()
                out = [tracker.update(p, b, c) for p, (b, c) in enumerate(frames)]
                if w:
                    host[key].append(time.perf_counter() - t0)
            if key == "sort_ref_route":
                ref_ids, ref_boxes = np.stack([o[0] for o in out]), np.stack([o[1] for o in out])
    nan = np.isnan(ref_boxes)
    equal = bool(np.array_equal(ids, ref_ids) and np.array_equal(np.isnan(boxes), nan) and
                 np.array_equal(np.where(nan, 0, boxes), np.where(nan, 0, ref_boxes)))
    dev = torch.device("cuda", plain.device_index)
    kernel = {"route": time_kernel(blocks, C, K, 1, batch, windows, dev),
              "dense_voc": time_kernel(dense, C, K, 1, batch, windows, dev),
              "coco_bound": time_kernel(bound_blocks(80, 100, n), 80, 100, 9, batch, windows, dev)}
    return {"frames_per_s": {k: round(n / statistics.median(v), 1) for k, v in times.items()},
            "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()},
            "track_kernel_ms_per_batch_median_max": kernel,
            "host_frames_per_s": {k: round(n / statistics.median(v), 1) for k, v in host.items()},
            "host_windows_s": {k: [round(t, 4) for t in v] for k, v in host.items()},
            "reported_records": int((ids >= 0).sum()), "tracks": int(ids.max(initial=0)), "ids_equal": equal}


def _same(ids, boxes, ref_ids, ref_boxes):
    nan = np.isnan(ref_boxes)
    return bool(np.array_equal(ids, ref_ids) and np.array_equal(np.isnan(boxes), nan) and
                np.array_equal(np.where(nan, 0, boxes).view(np.int32), np.where(nan, 0, ref_boxes).view(np.int32)))


def ocsort_bound_blocks(C, K, n):
    """``bound_blocks`` with a high score (0.9) on every record: class 0 is given K new boxes in every frame that overlap
    nothing, so that it holds K (max_age + 1) tracks."""
    return [(b, c, np.full((C, K), 0.9, np.float32)) for b, c in bound_blocks(C, K, n)]


def scored_trackers(method):
    """(obj_thresh of its pipelines, GPU tracker(C, K, device), host tracker(C, K), the bound stream's (C, K, blocks(n),
    tracker(device))) of the --track bytetrack / ocsort arms."""
    from k210_yolo_framework_b200.track import ByteTracker, OcSortTracker
    from oracle import bytetrack_ref, ocsort_ref
    if method == "bytetrack":
        return (0.1, lambda C, K, d: ByteTracker(C, K, device=d), bytetrack_ref.ByteTrack,
                (80, 100, lambda n: bytetrack_bound_blocks(80, 100, n), lambda d: ByteTracker(80, 100, device=d)))
    return (0.3, lambda C, K, d: OcSortTracker(C, K, device=d), ocsort_ref.OcSort,
            (80, 100, lambda n: ocsort_bound_blocks(80, 100, n), lambda d: OcSortTracker(80, 100, max_age=39, device=d)))


def bench_scored(make_pipe, n, load, batch, windows, method):
    """The --track bytetrack and --track ocsort arms (see the module docstring)."""
    obj_thresh, gpu_tracker, host_tracker, (bC, bK, bound, bound_tracker) = scored_trackers(method)
    plain, tracked = make_pipe(obj_thresh), make_pipe(obj_thresh)
    C, K = plain.gather.C, plain.gather.K
    recs = run(plain, n, load, 4)                                   # warm-up of both
    tracked.enable_tracking(method=method)
    got = []
    assert run(tracked, n, load, 4, tracks=got) == recs             # tracking leaves the records as they were
    times = {"gpu_plain": [], "gpu_track": []}
    for w in range(windows):
        arms = ["gpu_plain", "gpu_track"] if w % 2 == 0 else ["gpu_track", "gpu_plain"]
        for arm in arms:
            if arm == "gpu_track":
                tracked.reset_tracks()
                got = []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run(tracked, n, load, 4, tracks=got) if arm == "gpu_track" else run(plain, n, load, 4)
            torch.cuda.synchronize()
            times[arm].append(time.perf_counter() - t0)
            assert out == recs
    ids = torch.cat([g[0] for g in got]).numpy()
    boxes = torch.cat([g[1] for g in got]).numpy()
    blocks = frame_blocks(recs, C, K, scores=True)
    dense = with_scores(dense_voc_blocks(C, K, n))
    host, ref = {}, {}
    for stream, frames in (("route", blocks), ("dense_voc_first_batch", dense[:batch])):
        host[stream] = []
        for w in range(windows + 1):            # the first pass warms up
            tracker = host_tracker(C, K)
            t0 = time.perf_counter()
            out = [tracker.update(p, *f) for p, f in enumerate(frames)]
            if w:
                host[stream].append(time.perf_counter() - t0)
        ref[stream] = np.stack([o[0] for o in out]), np.stack([o[1] for o in out])
    dev = torch.device("cuda", plain.device_index)
    first = []
    kernel = {"route": time_kernel(blocks, C, K, 0, batch, windows, dev, lambda: gpu_tracker(C, K, dev.index)),
              "dense_voc": time_kernel(dense, C, K, 0, batch, windows, dev, lambda: gpu_tracker(C, K, dev.index), first),
              "coco_bound": time_kernel(bound(n), bC, bK, 0, batch, windows, dev, lambda: bound_tracker(dev.index))}
    equal = {"route": _same(ids, boxes, *ref["route"]), "dense_voc_first_batch": _same(*first, *ref["dense_voc_first_batch"])}
    return {"obj_thresh": obj_thresh, "records": int(sum(len(r) for r in recs)),
            "frames_per_s": {k: round(n / statistics.median(v), 1) for k, v in times.items()},
            "windows_s": {k: [round(t, 4) for t in v] for k, v in times.items()},
            f"{method}_kernel_ms_per_batch_median_max": kernel,
            f"{method}_ref_frames_per_s": {k: round(len(blocks if k == "route" else dense[:batch]) / statistics.median(v), 1)
                                           for k, v in host.items()},
            "reported_records": int((ids >= 0).sum()), "tracks": int(ids.max(initial=0)), "ids_equal_by_stream": equal,
            "ids_equal": all(equal.values())}


if __name__ == "__main__":
    main()
