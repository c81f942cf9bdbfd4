#!/usr/bin/env python
"""Batched serving front-end: a directory (or list) of images -> batches -> image-shard over the GPUs of the box ->
gathered detections, one JSON line per image.  The GPU analogue of the firmware's capture -> run -> draw loop
(/root/reference/yolo3_frame_test_public/main.c:294-326) and of calling keras_inference.py once per file.

    python serve.py CKPT IMAGE_DIR [--model_def yolo_mobilev1 --depth_multiplier 0.75 --image_size 224 320 --class_num 20
                                    --anchors data/voc_anchor.npy --batch 32 --obj_thresh 0.7 --iou_thresh 0.5 --out dets.jsonl]
    python -m torch.distributed.run --nproc-per-node 8 serve.py ...        # one rank per GPU, NCCL all-gather of the records
    python serve.py CKPT IMAGE_DIR --draw OUT_DIR [--draw_quality 75]       # also OUT_DIR/<stem>.jpg with the detections drawn

Per global batch of world*batch images: every rank reads ITS files in a pool of --decode_threads threads, one batch ahead.
Baseline JPEGs the GPU decoder takes (preprocess.gpu_decodable) stay compressed; every other file is decoded there by PIL as
Helper._read_img does.  DetectionPipeline.submit_images takes both (one packed H2D copy, the JPEG decode on the GPU, one
batched letterbox launch into its uint8 input buffer, network + decode + NMS), and ONE all-gather completes the record blocks
on every rank; two batches are in flight, and rank 0 writes the lines in file order.  The GPU decode gives the bytes PIL
gives, so the lines do not depend on which route a file took.

With --draw DIR every rank also writes DIR/<stem>.jpg for its own files: the records are drawn onto the original images where
they already lie on the GPU and encoded there (DetectionPipeline.enable_rendering), with the bytes PIL's draw_detections + save
give; only the compressed files come back.  Duplicate stems are refused before any work starts.

With --tiles ROWS COLS every image is detected on ROWS x COLS overlapping tiles as well as whole (--tile_overlap, default 0.2;
DetectionPipeline.enable_tiling): a batch then holds batch // (1 + ROWS * COLS) images, the views' records are merged on the GPU
and the lines keep their shape, with "index" // (boxes per network input) telling the view a detection came from.
--tile_size H W --tile_images N plans each image's grid from its own size instead (tiles of at most H x W pixels, a batch of N
images); --tile_match ios, --tile_merge union and --tile_border PX change how the views' records are merged (either grid).
With --flip every view (the whole image, or each of its tiles) is also detected mirrored left to right, the test-time
augmentation of a detector trained with random flips (DetectionPipeline.enable_flip): a batch then holds half the images, and the
mirrored views' records are mapped back and merged with the rest on the GPU.  It combines with every tiling flag.

With --gpu_png the PNG files the GPU decoder takes (preprocess.png_gpu_decodable) stay compressed too and are decoded on the GPU
(DetectionPipeline.enable_png_decode), with the pixels PIL gives; the lines are the same as without it.  --gpu_progressive does
the same for the progressive JPEGs the GPU decoder takes (preprocess.progressive_gpu_decodable,
DetectionPipeline.enable_progressive_jpeg_decode).

IMAGE_DIR may also be a video file, recognised by its content (RIFF AVI, MP4 / MOV, Matroska / WebM; video files inside a
directory are not picked up).  Its frames go through the same loop, one JSON line per frame in frame order,
{"video": PATH, "frame": i, "time": seconds, "detections": [...]}, and every flag works per frame.  Motion-JPEG frames in an AVI
are read by index (k210_yolo_framework_b200.video) and routed as JPEG files are; every other video is decoded in order by
OpenCV's FFmpeg backend on the decode threads of every rank, each rank keeping its own frames.  --draw DIR then writes
DIR/<stem>.avi, a Motion-JPEG AVI of the drawn frames at the source frame rate, on rank 0.

Several video files may be given at once (and only video files, each once): they are all served at the same time, their
frames interleaved in the same batches (``interleave``, one frame of each video in turn), so N camera recordings share one
pipeline and its batches instead of taking N runs.  Each video keeps its own lines, "video" naming it; the lines of
different videos interleave in batch order, and each video's lines stay in frame order.  --draw DIR writes one
DIR/<stem>.avi per video (two videos with one stem are refused before any work), and under --track each video is its own
stream (DetectionPipeline.enable_tracking(streams=...)), with its own ids from 1: every video's lines are those it gives
served alone.  One input behaves as it always has.

With --track (videos only) the objects are tracked across the frames on the GPU, SORT-style (DetectionPipeline.enable_tracking,
--track_max_age, --track_min_hits, --track_iou), or with --tracker bytetrack by ByteTrack (--track_thresh, --track_match,
--track_buffer, --track_no_fuse_score; its low-score association sees only the records above --obj_thresh, so it wants
--obj_thresh 0.1), or with --tracker ocsort by OC-SORT (--track_max_age, default 30, --track_min_hits, --track_iou,
--track_det_thresh, --track_delta_t, --track_inertia, --track_use_byte): every detection of a line gains "track", its track id
or null, and "track_box_tlbr", the track's box, when it has an id (under OC-SORT the record's own box).  Dropped frames count
as frames without detections.  With --track --draw DIR --draw_tracks each DIR/<stem>.avi shows the tracks instead of the
records (DetectionPipeline.enable_rendering(tracks=True), draw.draw_tracks): every track box in the colour of its id, labelled
"{class:2d} #{id}", so an id switch shows as a change of colour and label.  The JSON lines do not change.
"""
import argparse
import io
import json
import os
import sys
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from k210_yolo_framework_b200.dist import shard_range  # noqa: E402
from k210_yolo_framework_b200.helper import read_image  # noqa: E402
from k210_yolo_framework_b200.preprocess import gpu_decodable, png_gpu_decodable, progressive_gpu_decodable  # noqa: E402
from k210_yolo_framework_b200.pipeline import DetectionPipeline  # noqa: E402
from k210_yolo_framework_b200.video import AviWriter, jpeg_hw, open_video, sniff_video  # noqa: E402

EXTS = (".jpg", ".jpeg", ".png", ".bmp")


def list_images(path):
    if os.path.isdir(path):
        return sorted(os.path.join(path, f) for f in os.listdir(path) if f.lower().endswith(EXTS))
    with open(path) as fh:
        return [l.strip() for l in fh if l.strip()]


def is_video(path):
    """True when `path` is a file whose content is a video container (RIFF AVI, ISO-BMFF or Matroska / WebM); directories and
    text lists of images are not."""
    if not os.path.isfile(path):
        return False
    with open(path, "rb") as fh:
        return sniff_video(fh.read(12))


def route_image(data, gpu_png=False, gpu_progressive=False):
    """A file's bytes when the GPU decodes it (PNGs only with `gpu_png`, progressive JPEGs only with `gpu_progressive`), else
    its pixels decoded on the host (Helper._read_img)."""
    if gpu_decodable(data) or (gpu_png and png_gpu_decodable(data)) or (gpu_progressive and progressive_gpu_decodable(data)):
        return data
    return read_image(io.BytesIO(data))


def load_image(path, gpu_png=False, gpu_progressive=False):
    """``route_image`` of the file at `path`."""
    with open(path, "rb") as fh:
        return route_image(fh.read(), gpu_png, gpu_progressive)


def open_pipeline(args, max_per_class=30):
    """(pipe, world, rank): this rank's DetectionPipeline for the model / anchor / batch / threshold flags, after joining the
    process group when the job spans several GPUs (torch.distributed.run's environment)."""
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    anchors = np.load(args.anchors)
    pipe = DetectionPipeline(args.model_def, tuple(args.image_size), anchors, args.class_num, args.depth_multiplier, args.batch,
                             args.obj_thresh, args.iou_thresh, max_per_class, device=local, world=world, rank=rank)
    pipe.engine.load_weights(args.ckpt)
    options = dict(match=getattr(args, "tile_match", "iou"), merge=getattr(args, "tile_merge", "suppress"),
                   border=getattr(args, "tile_border", None))
    if getattr(args, "tiles", None):
        pipe.enable_tiling(args.tiles[0], args.tiles[1], args.tile_overlap, **options)
    elif getattr(args, "tile_size", None):
        pipe.enable_tiling(overlap=args.tile_overlap, tile_size=tuple(args.tile_size), images_per_batch=args.tile_images, **options)
    if getattr(args, "flip", False):
        pipe.enable_flip(**options)
    if getattr(args, "gpu_png", False):
        pipe.enable_png_decode()
    if getattr(args, "gpu_progressive", False):
        pipe.enable_progressive_jpeg_decode()
    return pipe, world, rank


def draw_paths(files, out_dir, ext=".jpg"):
    """``out_dir/<stem><ext>`` for every input file (.avi for videos); raises ValueError when two files share a stem (their
    drawn results would overwrite each other)."""
    seen = {}
    for p in files:
        stem = os.path.splitext(os.path.basename(p))[0]
        if stem in seen:
            raise ValueError(f"--draw: {seen[stem]} and {p} would both be written to {stem}{ext}")
        seen[stem] = p
    return [os.path.join(out_dir, os.path.splitext(os.path.basename(p))[0] + ext) for p in files]


def interleave(lengths, slots, G):
    """The schedule of sequences of `lengths` frames served through `slots` stream slots, G frames a global batch: a list with
    per global batch (frames, resets), `frames` the batch's (sequence, frame, slot) in row order and `resets` the slots to
    reset before it.  Round-robin: one frame per active sequence a turn, in slot order (the turns carry on from one batch
    to the next), until the batch holds G frames or no active sequence has frames left.  When a batch starts, each free
    slot, lowest first, takes the next sequence in the given order; a slot freed in a batch is taken again from the next
    batch only, after its reset, so two sequences never share a slot within a batch.  Sequences of no frames are skipped.
    So one slot runs the sequences one after another, each in batches of G frames with a short last one, and slots >=
    len(lengths) runs them all at once in full batches but the last."""
    slots, G = int(slots), int(G)
    if slots < 1 or G < 1:
        raise ValueError(f"{slots} slots and {G} frames a batch: both must be >= 1")
    todo = deque(i for i, n in enumerate(lengths) if n > 0)
    active, used = [None] * slots, [False] * slots      # per slot: [sequence, its next frame]; whether it ever held one
    left = lambda a: a is not None and a[1] < lengths[a[0]]
    out, turn = [], 0
    while todo or any(a is not None for a in active):
        resets = []
        for slot in range(slots):
            if active[slot] is None and todo:
                if used[slot]:
                    resets.append(slot)
                active[slot], used[slot] = [todo.popleft(), 0], True
        frames = []
        while len(frames) < G and any(left(a) for a in active):
            a = active[turn]
            if left(a):
                frames.append((a[0], a[1], turn))
                a[1] += 1
            turn = (turn + 1) % slots
        active = [a if left(a) else None for a in active]
        out.append((frames, resets))
    return out


def detect_files(pipe, files, decode_threads=4, load=None, rendered=False, positions=None, schedule=None):
    """Yields ``(paths, dets, counts)`` per global batch of world * images_per_batch files, in file order: the batch's gathered
    record blocks as ``collect`` returns them (pinned host views, valid until the generator resumes twice; with tiling on
    several ranks, copies of the rows that hold images, so that row j is file j here too).  Every rank reads ITS
    files of the next batch in a pool of `decode_threads` threads while the GPU works, and two batches are in flight.
    Every rank runs the network on a full batch (the tensor-core plans depend on the batch size, so the records of a short
    final batch match a full one's bit for bit) and takes part in every all-gather: its share of a short batch is padded
    with a grey network-size image, whose records nobody reads.  `load` maps a path to what submit_images takes
    (default: load_image).  With `rendered` (the pipeline's rendering enabled) each tuple also carries this rank's drawn
    JPEG files of the batch, its padding images' files left out.  With `positions` (the pipeline's tracking enabled; each
    file's position in the stream) the batch's positions go to submit_images and each tuple ends with ``pipe.tracks``: the
    (ids, boxes) of the batch's files, row j being file j.

    With `schedule` (``interleave``'s batches for G = world * images_per_batch) the frames of several sequences share the
    batches instead: `files` is not used, the keys (what `load` takes and the tuples list) are (sequence, frame) pairs,
    `positions[sequence][frame]` gives each frame's position, and with `positions` each frame's slot is its stream
    (submit_images' `streams`) and the batch's resets run before it is submitted (``reset_tracks(slot)``)."""
    load = load or load_image
    B, G, rank = pipe.images_per_batch, pipe.world * pipe.images_per_batch, pipe.rank
    rows = None
    if pipe.world > 1 and B != pipe.batch:      # rank r's B images lie from row r * batch of the gathered block
        rows = [r * pipe.batch + j for r in range(pipe.world) for j in range(B)]
    if schedule is None:
        chunks = [files[g0:g0 + G] for g0 in range(0, len(files), G)]
        plan = [(chunk, None if positions is None else {"frames": [positions[g * G + q] for q in range(len(chunk))]}, [])
                for g, chunk in enumerate(chunks)]
    else:
        plan = [([(i, k) for i, k, _ in frames], None if positions is None else
                 {"frames": [positions[i][k] for i, k, _ in frames], "streams": [slot for _, _, slot in frames]}, resets)
                for frames, resets in schedule]
        if any(len(chunk) > G for chunk, _, _ in plan):
            raise ValueError(f"a schedule batch holds more than the {G} frames of a global batch")
    filler = np.full(pipe.in_hw + (3,), 128, np.uint8)
    with ThreadPoolExecutor(max(1, int(decode_threads))) as pool:
        def decode(chunk):      # this rank's images of a global batch, decoding in the pool
            return [pool.submit(load, p) for p in chunk[rank * B:(rank + 1) * B]]

        def result(chunk, ticket, mine):
            dets, counts = pipe.collect(ticket)
            out = (chunk, dets, counts) if rows is None else (chunk, dets[rows], counts[rows])
            out = out + (pipe.rendered(ticket)[:mine],) if rendered else out
            return out + (pipe.tracks(ticket),) if positions is not None else out

        pending = deque()
        nxt = decode(plan[0][0]) if plan else []
        for g, (chunk, kw, resets) in enumerate(plan):
            imgs = [f.result() for f in nxt]
            nxt = decode(plan[g + 1][0]) if g + 1 < len(plan) else []
            if kw is not None:
                for slot in resets:
                    pipe.reset_tracks(slot)
            pending.append((chunk, pipe.submit_images(imgs + [filler] * (B - len(imgs)), **(kw or {})), len(imgs)))
            if len(pending) == 2:
                yield result(*pending.popleft())
        while pending:
            yield result(*pending.popleft())


def detections(recs, track=None):
    """The "detections" field of a JSON line: one image's (or frame's) records.  With `track` = (ids, boxes, counts) of the
    frame (``DetectionPipeline.tracks`` and the record counts) each detection also gets "track" (null without one) and, with
    an id, "track_box_tlbr"."""
    out = [{"class": int(c), "score": round(float(s), 6), "box_tlbr": [float(t), float(l), float(b), float(r)], "index": int(i)}
           for c, i, s, t, l, b, r in recs]
    if track is not None:
        ids, boxes, counts = (np.asarray(a) for a in track)
        mine = np.arange(ids.shape[1])[None, :] < counts[:, None]      # the records, class-major as `recs` lists them
        for d, tid, box in zip(out, ids[mine].tolist(), boxes[mine].tolist()):
            d["track"] = tid if tid >= 0 else None
            if tid >= 0:
                d["track_box_tlbr"] = box
    return out


def input_paths(args):
    """The input positional as a list (a single path given as a string is one input)."""
    return [args.images] if isinstance(args.images, str) else list(args.images)


def serve(args, out_fh=None):
    import torch.distributed as dist
    paths = input_paths(args)
    if is_video(paths[0]):
        return serve_video(args, out_fh)
    files = list_images(paths[0])
    draw_dir = getattr(args, "draw", None)
    targets = draw_paths(files, draw_dir) if draw_dir else None     # refuses duplicate stems before any work
    pipe, world, rank = open_pipeline(args)
    if draw_dir:
        os.makedirs(draw_dir, exist_ok=True)
        pipe.enable_rendering(quality=args.draw_quality)
    n_out = 0
    B = pipe.images_per_batch
    gpu_png, gpu_progressive = getattr(args, "gpu_png", False), getattr(args, "gpu_progressive", False)
    load = (lambda p: load_image(p, gpu_png, gpu_progressive)) if gpu_png or gpu_progressive else load_image
    for g, item in enumerate(detect_files(pipe, files, getattr(args, "decode_threads", 4), load, rendered=bool(draw_dir))):
        chunk, dets, counts = item[:3]
        if draw_dir:        # this rank's files of the global batch
            first = g * world * B + rank * B
            for path, data in zip(targets[first:first + len(item[3])], item[3]):
                with open(path, "wb") as fh:
                    fh.write(data)
        if rank != 0:
            continue
        recs = DetectionPipeline.records(dets, counts)
        for j, path in enumerate(chunk):
            line = {"image": path, "detections": detections(recs[j])}
            if out_fh is not None:
                out_fh.write(json.dumps(line) + "\n")
            n_out += 1
    if world > 1:
        dist.barrier()
    return n_out


def serve_video(args, out_fh=None):
    """``serve`` for one or more video files: one JSON line per frame, {"video", "frame" (its position in the stream), "time"
    (seconds), "detections"}, each video's lines in frame order.  Several videos share the batches (``interleave``, one slot
    and, under --track, one tracking stream per video), and the lines of different videos interleave in batch order.
    Frames are batched and sharded over the ranks as files are (``detect_files``); Motion-JPEG AVI frames are read by index
    and routed as image files are, other videos are decoded in order by OpenCV's FFmpeg backend on every rank, each keeping
    its own frames.  With --draw DIR rank 0 writes DIR/<stem>.avi per video at its source frame rate from the GPU-drawn JPEG
    frames, which the other ranks send it once per global batch."""
    import torch.distributed as dist
    paths = input_paths(args)
    draw_dir = getattr(args, "draw", None)
    targets = draw_paths(paths, draw_dir, ".avi") if draw_dir else None      # refuses duplicate stems before any work
    srcs = [open_video(p) for p in paths]
    pipe, world, rank = open_pipeline(args)
    if draw_dir:
        os.makedirs(draw_dir, exist_ok=True)
        pipe.enable_rendering(quality=args.draw_quality, tracks=getattr(args, "draw_tracks", False))
    track = getattr(args, "track", False)
    if track:
        enable_tracking(pipe, args, streams=len(srcs))
    B, G = pipe.images_per_batch, pipe.world * pipe.images_per_batch
    schedule = interleave([src.n_frames for src in srcs], len(srcs), G)
    mine = {(i, k) for frames, _ in schedule for q, (i, k, _) in enumerate(frames) if q // B == rank}   # this rank's frames
    gpu_png, gpu_progressive = getattr(args, "gpu_png", False), getattr(args, "gpu_progressive", False)
    loads = [src.loader(keep=lambda k, i=i: (i, k) in mine, route=lambda data: route_image(data, gpu_png, gpu_progressive))
             for i, src in enumerate(srcs)]
    writers, n_out = [None] * len(srcs), 0
    try:
        positions = [[src.position(k) for k in range(src.n_frames)] for src in srcs] if track else None
        for item in detect_files(pipe, None, getattr(args, "decode_threads", 4), lambda key: loads[key[0]](key[1]),
                                 rendered=bool(draw_dir), positions=positions, schedule=schedule):
            chunk, dets, counts = item[:3]
            if draw_dir:
                drawn = item[3]
                if world > 1:       # the frames vary in size: the records' fixed-size all-gather cannot carry them
                    parts = [None] * world if rank == 0 else None
                    dist.gather_object(drawn, parts, dst=0)
                    drawn = [d for part in parts for d in part] if rank == 0 else []
                for (i, _), data in zip(chunk, drawn):
                    if writers[i] is None:
                        writers[i] = AviWriter(targets[i], srcs[i].fps, jpeg_hw(data))
                    writers[i].write(data)
            if rank != 0:
                continue
            recs = DetectionPipeline.records(dets, counts)
            for j, (i, k) in enumerate(chunk):
                tr = (item[-1][0][j], item[-1][1][j], counts[j]) if track else None
                line = {"video": paths[i], "frame": srcs[i].position(k), "time": srcs[i].time(k), "detections": detections(recs[j], tr)}
                if out_fh is not None:
                    out_fh.write(json.dumps(line) + "\n")
                n_out += 1
    finally:
        for w in writers:
            if w is not None:
                w.close()
    if world > 1:
        dist.barrier()
    return n_out


def add_model_args(ap):
    """The model, anchor, batch and decode-thread flags serve.py and evaluate_map.py share."""
    ap.add_argument("ckpt")
    ap.add_argument("--model_def", default="yolo_mobilev1", choices=["yolo_mobilev1", "yolo_mobilev2", "tiny_yolo", "yolo"])
    ap.add_argument("--depth_multiplier", type=float, default=0.75)
    ap.add_argument("--image_size", type=int, nargs=2, default=(224, 320))
    ap.add_argument("--class_num", type=int, default=20)
    ap.add_argument("--anchors", default="data/voc_anchor.npy")
    ap.add_argument("--batch", type=int, default=32, help="images per GPU per step")
    grid = ap.add_mutually_exclusive_group()
    grid.add_argument("--tiles", type=int, nargs=2, default=None, metavar=("ROWS", "COLS"),
                      help="also detect on ROWS x COLS overlapping tiles of every image and merge the views' records on the GPU; "
                           "a batch then holds batch // (1 + ROWS * COLS) images")
    grid.add_argument("--tile_size", type=int, nargs=2, default=None, metavar=("H", "W"),
                      help="also detect on overlapping tiles of at most H x W pixels, as many as each image's size needs (an "
                           "image that fits one tile is detected whole only); needs --tile_images")
    ap.add_argument("--tile_images", type=int, default=None, metavar="N",
                    help="images per batch with --tile_size; each image gets at most batch // N views")
    ap.add_argument("--tile_overlap", type=float, default=0.2, help="fraction of a tile shared with its neighbour (with --tiles)")
    ap.add_argument("--tile_match", choices=["iou", "ios"], default="iou",
                    help="merge views' records matching by IoU or by intersection over the smaller box (threshold --iou_thresh)")
    ap.add_argument("--tile_merge", choices=["suppress", "union"], default="suppress",
                    help="drop a matching record, or also grow the kept record's box to the union of the records it suppressed")
    ap.add_argument("--tile_border", type=float, default=None, metavar="PX",
                    help="drop a tile's records within PX pixels of a tile edge inside the image before the merge")
    ap.add_argument("--flip", action="store_true",
                    help="also detect every view mirrored left to right and merge both on the GPU (a batch holds half the images)")
    ap.add_argument("--gpu_png", action="store_true",
                    help="decode the PNG files the GPU decoder takes on the GPU too (the same pixels as PIL), not in the host threads")
    ap.add_argument("--gpu_progressive", action="store_true",
                    help="decode the progressive JPEG files the GPU decoder takes on the GPU too (the same pixels as PIL), not in "
                         "the host threads")
    ap.add_argument("--decode_threads", type=int, default=4, help="host threads reading the next batch's files and decoding those the GPU does not (PIL)")


class ModelArgParser(argparse.ArgumentParser):
    """An ArgumentParser that also refuses the add_model_args flags that need one another alone: --tile_size without
    --tile_images, and --tile_images without --tile_size; and, with add_track_args, the flags of the tracker --tracker does
    not select."""

    def parse_known_args(self, args=None, namespace=None):
        ns, rest = super().parse_known_args(args, namespace)
        size, n = getattr(ns, "tile_size", None), getattr(ns, "tile_images", None)
        if size is not None and n is None:
            self.error("--tile_size needs --tile_images N: the images one batch holds")
        if n is not None and size is None:
            self.error("--tile_images goes with --tile_size")
        if hasattr(ns, "tracker"):
            fill_track_defaults(ns)
            if track_args_error(ns):
                self.error(track_args_error(ns))
        return ns, rest


def quality_arg(v):
    q = int(v)
    if not 1 <= q <= 100:
        raise argparse.ArgumentTypeError(f"JPEG quality {v} is outside 1..100")
    return q


class ServeArgParser(ModelArgParser):
    """serve.py's parser: also refuses --track for anything but video files, several inputs unless all are video files, the
    same input twice, with --draw two videos of one stem, and --draw_tracks without --track and --draw."""

    def parse_known_args(self, args=None, namespace=None):
        ns, rest = super().parse_known_args(args, namespace)
        paths = input_paths(ns)
        if len(paths) > 1:
            if len({os.path.realpath(p) for p in paths}) < len(paths):
                self.error("the same input is given twice")
            others = [p for p in paths if not is_video(p)]
            if others:
                self.error(f"several inputs must all be video files; {others[0]} is not")
            if getattr(ns, "draw", None):
                try:
                    draw_paths(paths, ns.draw, ".avi")
                except ValueError as e:
                    self.error(str(e))
        if getattr(ns, "track", False) and not is_video(paths[0]):
            self.error(f"--track tracks the frames of a video; {paths[0]} is not a video file")
        if getattr(ns, "draw_tracks", False) and not (getattr(ns, "track", False) and getattr(ns, "draw", None)):
            self.error("--draw_tracks draws the tracks into the --draw videos: it needs --track and --draw")
        return ns, rest


def build_parser():
    ap = ServeArgParser()
    add_model_args(ap)
    ap.add_argument("images", nargs="+", metavar="IMAGES",
                    help="directory of images, a text file with one path per line, or one or more video files (recognised by "
                         "their content: AVI, MP4 / MOV or Matroska / WebM), served together")
    ap.add_argument("--obj_thresh", type=float, default=0.7)
    ap.add_argument("--iou_thresh", type=float, default=0.5)
    ap.add_argument("--out", default="-")
    ap.add_argument("--draw", default=None, metavar="DIR",
                    help="also write every image with its detections drawn (as keras_inference.py draws them) to DIR/<stem>.jpg, "
                         "rendered and JPEG-encoded on the GPU; for a video, its drawn frames as the Motion-JPEG AVI DIR/<stem>.avi")
    ap.add_argument("--draw_quality", type=quality_arg, default=75, help="JPEG quality of the --draw files (1..100)")
    ap.add_argument("--track", action="store_true",
                    help="track objects across a video's frames on the GPU (SORT, or --tracker bytetrack or ocsort): each "
                         "detection gains its track id and box")
    add_track_args(ap, " (--track)")
    ap.add_argument("--draw_tracks", action="store_true",
                    help="draw the tracks into the --draw videos instead of the detections: each track box in its id's colour, "
                         "labelled with class and id (needs --track and --draw)")
    return ap


def add_track_args(ap, note=""):
    """The tracker flags serve.py and evaluate_mot.py share (DetectionPipeline.enable_tracking).  --track_max_age,
    --track_min_hits and --track_iou default to the selected tracker's values (ModelArgParser fills them in)."""
    ap.add_argument("--tracker", choices=["sort", "bytetrack", "ocsort"], default="sort",
                    help="SORT; ByteTrack, which also associates the tracks left with the low-score records (it sees only "
                         "the records above --obj_thresh, so its second association needs --obj_thresh 0.1); or OC-SORT, which "
                         "re-updates a re-found track along a virtual path, adds a direction term to the association and "
                         "re-matches by the tracks' last observations" + note)
    ap.add_argument("--track_max_age", type=int, default=None,
                    help="frames a track may miss before it is removed (SORT, default 1; OC-SORT, default 30)" + note)
    ap.add_argument("--track_min_hits", type=int, default=None,
                    help="matched frames in a row before a track is reported (SORT and OC-SORT, default 3)" + note)
    ap.add_argument("--track_iou", type=float, default=None,
                    help="least IoU of a detection with its track's prediction (SORT and OC-SORT, default 0.3)" + note)
    ap.add_argument("--track_thresh", type=float, default=0.5,
                    help="score above which a record is high (ByteTrack; low records score in (0.1, track_thresh))" + note)
    ap.add_argument("--track_match", type=float, default=0.8, help="largest cost of the first association (ByteTrack)" + note)
    ap.add_argument("--track_buffer", type=int, default=30, help="frames a lost track is kept (ByteTrack)" + note)
    ap.add_argument("--track_no_fuse_score", action="store_true",
                    help="associate by IoU alone, not IoU times score (ByteTrack; its --mot20)" + note)
    ap.add_argument("--track_det_thresh", type=float, default=0.6,
                    help="score above which a record is associated first and may start a track (OC-SORT)" + note)
    ap.add_argument("--track_delta_t", type=int, default=3,
                    help="frames back to the observation a track's direction is taken from, 1..8 (OC-SORT)" + note)
    ap.add_argument("--track_inertia", type=float, default=0.2, help="weight of the direction term (OC-SORT)" + note)
    ap.add_argument("--track_use_byte", action="store_true",
                    help="also associate the tracks left with the records scored in (0.1, track_det_thresh), as ByteTrack "
                         "does; it needs --obj_thresh 0.1 (OC-SORT)" + note)


SORT_FLAGS = {"track_max_age": 1, "track_min_hits": 3, "track_iou": 0.3}
BYTETRACK_FLAGS = {"track_thresh": 0.5, "track_match": 0.8, "track_buffer": 30, "track_no_fuse_score": False}
OCSORT_FLAGS = {"track_det_thresh": 0.6, "track_delta_t": 3, "track_inertia": 0.2, "track_use_byte": False}
OCSORT_SHARED = {"track_max_age": 30, "track_min_hits": 3, "track_iou": 0.3}


def fill_track_defaults(ns):
    """Gives --track_max_age, --track_min_hits and --track_iou, where left out, the value of the tracker --tracker selects."""
    for k, v in (OCSORT_SHARED if ns.tracker == "ocsort" else SORT_FLAGS).items():
        if getattr(ns, k) is None:
            setattr(ns, k, v)


def track_args_error(ns):
    """The message for add_track_args flags of the trackers --tracker does not select, set away from their defaults; None
    when there are none."""
    other = {"sort": {**BYTETRACK_FLAGS, **OCSORT_FLAGS}, "bytetrack": {**SORT_FLAGS, **OCSORT_FLAGS},
             "ocsort": BYTETRACK_FLAGS}[ns.tracker]
    wrong = [f"--{k}" for k, v in other.items() if getattr(ns, k) != v]
    if wrong:
        return f"{', '.join(wrong)} set another tracker than --tracker {ns.tracker}"
    return None


def enable_tracking(pipe, args, streams=1):
    """DetectionPipeline.enable_tracking with the add_track_args flags, for `streams` streams."""
    pipe.enable_tracking(args.track_max_age, args.track_min_hits, args.track_iou, method=args.tracker,
                         track_thresh=args.track_thresh, match_thresh=args.track_match, track_buffer=args.track_buffer,
                         fuse_score=not args.track_no_fuse_score, det_thresh=args.track_det_thresh,
                         delta_t=args.track_delta_t, inertia=args.track_inertia, use_byte=args.track_use_byte, streams=streams)


def main():
    args = build_parser().parse_args()
    rank = int(os.environ.get("RANK", "0"))
    fh = (sys.stdout if args.out == "-" else open(args.out, "w")) if rank == 0 else None
    n = serve(args, fh)
    if rank == 0 and fh is not sys.stdout:
        fh.close()
        print(f"{n} {'frames' if is_video(input_paths(args)[0]) else 'images'} -> {args.out}", file=sys.stderr)


if __name__ == "__main__":
    main()
