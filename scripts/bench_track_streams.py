#!/usr/bin/env python
"""Multi-stream tracking on one GPU: one launch of S streams against S single-stream launches of the same frames, and
several videos served together against one at a time.  Prints one JSON line.

    python scripts/bench_track_streams.py [--streams 1 8 32 132 264 --frames 32 --windows 3 --videos 96 64 128 --batch 32]

Kernel arm: S seeded dense streams (bench_video's "dense_voc": 20 classes, about 27 of 30 records each per frame; scored
as for ByteTrack and OC-SORT, 0.9 or 0.3; a different seed per stream) through each tracker at its default setting, 32
frames of every stream in one launch of a ``streams=S`` tracker, the frames of the streams taking turns in the batch.  In
the same run the same frames go through S single-stream trackers, one launch of 32 frames each: what tracking S feeds
takes without multi-stream tracking.  Each is timed from CUDA events over the whole set of launches, after one warm-up
pass, as the median of --windows passes: ms per S-stream batch and frames/s.  The outputs must be bit-identical between
the two, and stream 0 and the last stream must equal the oracle (oracle/sort_ref.py, bytetrack_ref.py, ocsort_ref.py) on
their first batch; the run fails otherwise.

Route arm: --videos synthetic 720p Motion-JPEG AVIs of uneven lengths (bench_video's frames, each video shifted) through
serve.py's serve_video with --track (SORT), all at once (one stream each) against one video at a time; frames/s over the
videos' frames, and each video's lines must be the same both ways.  The card's name and power limit are read in the run.
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

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import serve  # noqa: E402
from bench_ingest import GOLDEN, gpu_info  # noqa: E402
from bench_video import dense_voc_blocks, frames_720p, strip_dht, with_scores  # noqa: E402
from k210_yolo_framework_b200.dist import DetectionGather  # noqa: E402
from k210_yolo_framework_b200.track import ByteTracker, OcSortTracker, Tracker  # noqa: E402
from oracle import bytetrack_ref, ocsort_ref, sort_ref  # noqa: E402

C, K = 20, 30
TRACKERS = {"sort": (Tracker, lambda: sort_ref.Sort(C, K)), "bytetrack": (ByteTracker, lambda: bytetrack_ref.ByteTrack(C, K)),
            "ocsort": (OcSortTracker, lambda: ocsort_ref.OcSort(C, K))}


def stage(frames, dev):
    """The frames (boxes, counts, scores) as one gather block on the device, frame i in row i."""
    buf = torch.zeros((len(frames), C * (K * 6 + 1)), dtype=torch.int32)
    d, c = DetectionGather.split(buf, C, K)
    for i, (b, n, s) in enumerate(frames):
        d[i, :, :, :4] = torch.from_numpy(b.view(np.int32))
        d[i, :, :, 4] = torch.from_numpy(s.view(np.int32))
        c[i] = torch.from_numpy(n)
    return DetectionGather.split(buf.to(dev), C, K)


def timed(launch, reset, windows):
    """Median ms of `launch` over `windows` passes after one warm-up, each after `reset`, from CUDA events."""
    st = torch.cuda.current_stream()
    ms = []
    for w in range(windows + 1):
        reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        launch()
        b.record(st)
        torch.cuda.synchronize()
        if w:
            ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def kernel_arm(method, all_streams, S, F, windows, dev, oracle_cache):
    cls, oracle = TRACKERS[method]
    streams = all_streams[:S]
    st = torch.cuda.current_stream()
    # the multi-stream batch: frame f of every stream, then frame f + 1, ...
    order = [(s, f) for f in range(F) for s in range(S)]
    dets, counts = stage([streams[s][f] for s, f in order], dev)
    n = len(order)
    rows = torch.arange(n, dtype=torch.int32, device=dev)
    pos = torch.tensor([f for _, f in order], dtype=torch.int64, device=dev)
    strm = torch.tensor([s for s, _ in order], dtype=torch.int32, device=dev)
    ids, boxes = torch.empty((n, C, K), dtype=torch.int32, device=dev), torch.empty((n, C, K, 4), dtype=torch.float32, device=dev)
    multi = cls(C, K, device=dev.index, streams=S)
    last = {s: F - 1 for s in range(S)}
    ms_multi = timed(lambda: multi.update(dets, counts, rows, pos, n, ids, boxes, st, last, strm), multi.reset, windows)
    # S single-stream trackers, one launch of each stream's F frames
    blocks = [stage(streams[s], dev) for s in range(S)]
    singles = [cls(C, K, device=dev.index) for _ in range(S)]
    rows1, pos1 = torch.arange(F, dtype=torch.int32, device=dev), torch.arange(F, dtype=torch.int64, device=dev)
    ids1 = torch.empty((S, F, C, K), dtype=torch.int32, device=dev)
    boxes1 = torch.empty((S, F, C, K, 4), dtype=torch.float32, device=dev)

    def launch_singles():
        for s in range(S):
            singles[s].update(*blocks[s], rows1, pos1, F, ids1[s], boxes1[s], st, F - 1)

    def reset_singles():
        for t in singles:
            t.reset()

    ms_single = timed(launch_singles, reset_singles, windows)
    got_ids = ids.view(F, S, C, K).transpose(0, 1).cpu().numpy()
    got_boxes = boxes.view(F, S, C, K, 4).transpose(0, 1).cpu().numpy()
    one_ids, one_boxes = ids1.cpu().numpy(), boxes1.cpu().numpy()
    equal = bool(np.array_equal(got_ids, one_ids) and np.array_equal(got_boxes.view(np.int32), one_boxes.view(np.int32)))
    oracle_equal = True
    for s in sorted({0, S - 1}):
        if (method, s) not in oracle_cache:
            o = oracle()
            oracle_cache[method, s] = [o.update(f, b, c) if method == "sort" else o.update(f, b, c, sc)
                                       for f, (b, c, sc) in enumerate(streams[s])]
        for f, r in enumerate(oracle_cache[method, s]):
            oracle_equal &= bool(np.array_equal(r[0], got_ids[s, f]) and np.array_equal(
                np.asarray(r[1], np.float32).view(np.int32), got_boxes[s, f].view(np.int32)))
    frames = S * F
    return {"streams": S, "frames": frames, "ms_per_launch": round(ms_multi, 3), "frames_per_s": round(frames / ms_multi * 1e3, 1),
            "single_stream_ms": round(ms_single, 3), "single_stream_frames_per_s": round(frames / ms_single * 1e3, 1),
            "speedup": round(ms_single / ms_multi, 2), "outputs_equal": equal, "oracle_equal_first_batch": oracle_equal}


def make_videos(tmp, lengths):
    from PIL import Image
    pixels = frames_720p(max(lengths) + 7 * len(lengths))
    paths = []
    for v, n in enumerate(lengths):
        p = os.path.join(tmp, f"cam{v}.avi")
        with serve.AviWriter(p, 30.0, pixels[0].shape[:2]) as aw:
            for f in pixels[7 * v:7 * v + n]:
                b = io.BytesIO()
                Image.fromarray(f).save(b, "JPEG", quality=90, subsampling=1)
                aw.write(strip_dht(b.getvalue()))
        paths.append(p)
    return paths


def route_arm(lengths, batch, tmp):
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    from k210_yolo_framework_b200.yolonet import load_npz_weights
    ckpt = os.path.join(tmp, "model.h5")
    save_keras_weights(ckpt, load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    paths = make_videos(tmp, lengths)

    def serve_lines(videos):
        args = serve.build_parser().parse_args([ckpt] + videos + ["--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch",
                                                                  str(batch), "--obj_thresh", "0.3", "--track"])
        out = io.StringIO()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        serve.serve_video(args, out)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [json.loads(l) for l in out.getvalue().splitlines()]

    serve_lines(paths[:1])                      # warm-up: module loads, plans
    t_all, together = serve_lines(paths)
    t_one, equal = 0.0, True
    for p in paths:
        t, alone = serve_lines([p])
        t_one += t
        equal &= [l for l in together if l["video"] == p] == alone
    frames = sum(lengths)
    return {"videos": lengths, "batch": batch, "together_s": round(t_all, 3), "together_frames_per_s": round(frames / t_all, 1),
            "one_at_a_time_s": round(t_one, 3), "one_at_a_time_frames_per_s": round(frames / t_one, 1), "lines_equal": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 8, 32, 132, 264])
    ap.add_argument("--frames", type=int, default=32, help="frames of every stream in one launch")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--trackers", nargs="+", default=["sort", "bytetrack", "ocsort"], choices=sorted(TRACKERS))
    ap.add_argument("--videos", type=int, nargs="*", default=[96, 64, 128], help="frames of each video of the route arm")
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    out = {"gpu": gpu_info(), "kernel": {}}
    all_streams = [with_scores(dense_voc_blocks(C, K, args.frames, seed=s), seed=1000 + s) for s in range(max(args.streams))]
    cache = {}
    for method in args.trackers:
        out["kernel"][method] = [kernel_arm(method, all_streams, S, args.frames, args.windows, dev, cache) for S in args.streams]
    if args.videos:
        with tempfile.TemporaryDirectory() as tmp:
            out["route"] = route_arm(args.videos, args.batch, tmp)
    print(json.dumps(out))
    ok = all(r["outputs_equal"] and r["oracle_equal_first_batch"] for rs in out["kernel"].values() for r in rs)
    if not ok or not out.get("route", {"lines_equal": True})["lines_equal"]:
        sys.exit("outputs differ")


if __name__ == "__main__":
    main()
