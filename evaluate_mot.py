#!/usr/bin/env python
"""A checkpoint's tracking on MOTChallenge sequences: CLEAR MOT, the identity metrics and HOTA per sequence and combined,
with the tracking (SORT, ByteTrack with --tracker bytetrack or OC-SORT with --tracker ocsort: DetectionPipeline.enable_tracking) and the matching and counting on the GPU (evaluate.MotEval).

    python evaluate_mot.py CKPT SEQ [SEQ ...] --person_class N [--benchmark MOT17 --track_max_age 1 --track_min_hits 3
                                                                --track_iou 0.3 --results DIR --out mot.json]
    python evaluate_mot.py CKPT SEQ [SEQ ...] --person_class N --tracker bytetrack --obj_thresh 0.1 [--track_thresh 0.5
                                      --track_match 0.8 --track_buffer 30 --track_no_fuse_score ...]
    python evaluate_mot.py CKPT SEQ [SEQ ...] --person_class N --tracker ocsort [--track_max_age 30 --track_min_hits 3
                                      --track_iou 0.3 --track_det_thresh 0.6 --track_delta_t 3 --track_inertia 0.2
                                      --track_use_byte --obj_thresh 0.1 ...]
    python -m torch.distributed.run --nproc-per-node 8 evaluate_mot.py ...   # one rank per GPU; rank 0 evaluates

--streams N tracks up to N sequences at once, their frames interleaved in the same batches (serve.interleave; each in its
own tracking stream, DetectionPipeline.enable_tracking(streams=N)); the default 1 tracks them one after another.  The
tables, --out and --results are the same for every N.  N is a memory choice: each stream holds the tracker's state,
k2y_*_state_bytes() on the device, at the default settings per stream

                      VOC (C 20, K 30)    COCO (C 80, K 100)
    SORT                    0.3 MB                4.0 MB
    ByteTrack              10.4 MB              138.5 MB
    OC-SORT                21.8 MB              429.0 MB

(MB of 10^6 bytes; OC-SORT's K x cap scratch of round 1's costs per class makes it the largest, and --track_max_age or
--max_per_class shrink it).

SEQ is a MOTChallenge sequence directory (seqinfo.ini, imDir/%06d<imExt>, gt/gt.txt); a directory without seqinfo.ini
stands for its subdirectories that have one, sorted by name (such as MOT17/train).  Each sequence is one stream of frame
positions 0..seqLength-1, tracked from a fresh start.  A missing frame file, or one whose size differs from seqinfo.ini's,
raises ValueError.  --person_class is the network's class index that MOTChallenge calls pedestrian (14 for VOC, 0 for COCO);
its records with a track id are the tracker's rows: frame = position + 1, the track id, and the track box as (left, top, w,
h) with left = xmin + 1 and top = ymin + 1 (MOTChallenge pixels start at 1), in float64.

The protocol is TrackEval's MotChallenge2DBox with its CLEAR, Identity and HOTA metrics, as oracle/mot_ref.py and
oracle/mot_hota_ref.py restate them (not compared with TrackEval itself).  The first table holds CLEAR and Identity; the
second HOTA, DetA, AssA, DetRe, DetPr, AssRe, AssPr, LocA and OWTA, each the mean over the 19 alphas 0.05 .. 0.95 as
TrackEval's summary shows it, and HOTA(0), LocA(0) and HOTALocA(0).  --out writes both, the HOTA fields per alpha.  --results DIR writes DIR/<name>.txt in MOTChallenge tracker format, floats written with
repr so that reading a file back gives the evaluated values.  Sequences without gt/gt.txt are tracked and written with
--results but left out of the metrics.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from evaluate_map import load_checked  # noqa: E402
from serve import ModelArgParser, add_model_args, add_track_args, detect_files, enable_tracking, interleave, open_pipeline  # noqa: E402
from k210_yolo_framework_b200.evaluate import MOT_BENCHMARKS, MotEval, load_mot_gt, read_seqinfo  # noqa: E402

HOTA_COLUMNS = ("HOTA", "DetA", "AssA", "DetRe", "DetPr", "AssRe", "AssPr", "LocA", "OWTA", "HOTA(0)", "LocA(0)",
                "HOTALocA(0)")
COLUMNS = ("MOTA", "MOTP", "IDF1", "IDP", "IDR", "Rcll", "Prcn", "TP", "FP", "FN", "IDSW", "Frag", "MT", "PT", "ML", "IDTP",
           "IDFP", "IDFN")


def find_sequences(paths):
    """The sequence directories of the command line, in order; a directory without seqinfo.ini gives its subdirectories with
    one, sorted by name."""
    out = []
    for p in paths:
        if os.path.isfile(os.path.join(p, "seqinfo.ini")):
            out.append(p)
            continue
        subs = sorted(os.path.join(p, d) for d in os.listdir(p) if os.path.isfile(os.path.join(p, d, "seqinfo.ini"))) \
            if os.path.isdir(p) else []
        if not subs:
            raise ValueError(f"{p}: neither a sequence directory (seqinfo.ini) nor a directory of sequences")
        out += subs
    return out


def tracker_rows(positions, ids, boxes, dets, counts, person_class):
    """float64 [n, 7] (frame, id, left, top, w, h, conf) of a batch's tracked records of `person_class`, in record order."""
    ids, boxes, counts = np.asarray(ids), np.asarray(boxes, np.float32), np.asarray(counts)
    score = np.ascontiguousarray(np.asarray(dets)[:, person_class, :, 4]).view(np.float32)
    K = ids.shape[2]
    take = (np.arange(K)[None, :] < counts[:, person_class, None]) & (ids[:, person_class] >= 0)
    n, k = np.nonzero(take)
    b = boxes[n, person_class, k].astype(np.float64)
    frame = np.asarray(positions, np.float64)[n] + 1
    return np.stack([frame, ids[n, person_class, k].astype(np.float64), b[:, 1] + 1.0, b[:, 0] + 1.0, b[:, 3] - b[:, 1],
                     b[:, 2] - b[:, 0], score[n, k].astype(np.float64)], 1).reshape(-1, 7)


def write_results(path, rows):
    with open(path, "w") as fh:
        for r in rows.tolist():
            fh.write(f"{int(r[0])},{int(r[1])},{r[2]!r},{r[3]!r},{r[4]!r},{r[5]!r},{r[6]!r},-1,-1,-1\n")


def evaluate(args):
    """MotEval's result dict on rank 0 (None without any gt), None on the other ranks."""
    import torch.distributed as dist
    seqs = []
    for d in find_sequences(args.seqs):
        info = read_seqinfo(d)
        gt_path = os.path.join(d, "gt", "gt.txt")
        files = [os.path.join(d, info["imDir"], f"{k + 1:06d}{info['imExt']}") for k in range(info["seqLength"])]
        missing = [f for f in files if not os.path.isfile(f)]
        if missing:
            raise ValueError(f"{info['name']}: frame file {missing[0]} is missing")
        seqs.append((info, files, gt_path if os.path.isfile(gt_path) else None))
    if not any(s[2] for s in seqs) and not args.results:
        raise ValueError("no sequence has gt/gt.txt and --results is not given: nothing to do")
    pipe, world, rank = open_pipeline(args, args.max_per_class)
    if not 0 <= args.person_class < args.class_num:
        raise ValueError(f"--person_class {args.person_class} is outside [0, {args.class_num})")
    enable_tracking(pipe, args, streams=args.streams)
    ev = MotEval(args.benchmark, device=pipe.device_index) if rank == 0 and any(s[2] for s in seqs) else None
    if args.results and rank == 0:
        os.makedirs(args.results, exist_ok=True)
    if ev is not None:
        for info, _, gt_path in seqs:
            if gt_path:
                ev.add_sequence(info["name"], load_mot_gt(gt_path, args.benchmark), info["seqLength"])
    gpu_png, gpu_progressive = getattr(args, "gpu_png", False), getattr(args, "gpu_progressive", False)
    lengths = [info["seqLength"] for info, _, _ in seqs]
    schedule = interleave(lengths, args.streams, pipe.world * pipe.images_per_batch)
    rows = [[] for _ in seqs]
    loads = [(lambda k, f=files, hw=(info["imHeight"], info["imWidth"]): load_checked(f[k], hw, gpu_png, gpu_progressive))
             for info, files, _ in seqs]
    for chunk, dets, counts, (ids, boxes) in detect_files(pipe, None, args.decode_threads, lambda key: loads[key[0]](key[1]),
                                                          positions=[list(range(L)) for L in lengths], schedule=schedule):
        if rank != 0:
            continue
        for i in sorted({i for i, _ in chunk}):       # the batch's rows split by sequence, each in frame order
            (info, _, gt_path), js = seqs[i], [j for j, (q, _) in enumerate(chunk) if q == i]
            pos = [chunk[j][1] for j in js]
            part = [t[js] for t in (ids, boxes, dets, counts)]
            if ev is not None and gt_path:
                ev.update(info["name"], pos, *part, args.person_class)
            if args.results:
                rows[i].append(tracker_rows(pos, *part, args.person_class))
    if args.results and rank == 0:
        for (info, _, _), r in zip(seqs, rows):
            write_results(os.path.join(args.results, info["name"] + ".txt"), np.concatenate(r + [np.zeros((0, 7))]))
    if world > 1:
        dist.barrier()
    return ev.result() if ev is not None else None


def _table(rows, columns):
    fmt = (lambda v: f"{v:.4f}" if isinstance(v, float) else str(v))
    table = [["sequence"] + list(columns)] + [[n] + [fmt(d[k]) for k in columns] for n, d in rows]
    width = [max(len(r[i]) for r in table) for i in range(len(table[0]))]
    return "\n".join("  ".join(v.rjust(w) for v, w in zip(r, width)) for r in table)


def hota_summary(d):
    """TrackEval's summary of one HOTA dict: each per-alpha field's mean over the 19 alphas, and the (0) scalars."""
    out = {k: float(np.mean(d[k])) for k in HOTA_COLUMNS[:9]}
    out.update({k: d[k] for k in HOTA_COLUMNS[9:]})
    return out


def report(res):
    """One row per sequence and a COMBINED row of CLEAR and Identity; then the same rows of HOTA (means over alphas)."""
    rows = [(n, d) for n, d in res["sequences"].items()] + [("COMBINED", res["combined"])]
    text = _table(rows, COLUMNS)
    if "hota" in res:
        h = res["hota"]
        rows = [(n, hota_summary(d)) for n, d in h["sequences"].items()] + [("COMBINED", hota_summary(h["combined"]))]
        text += "\n\n" + _table(rows, HOTA_COLUMNS)
    return text


def to_json(res):
    return {"sequences": res["sequences"], "combined": res["combined"], "hota": res["hota"]}


def streams_arg(v):
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"--streams {v}: at least 1")
    return n


def build_parser():
    ap = ModelArgParser()
    add_model_args(ap)
    ap.add_argument("seqs", nargs="+", metavar="SEQ", help="MOTChallenge sequence directory, or a directory of them")
    ap.add_argument("--person_class", type=int, required=True,
                    help="the network's class index MOTChallenge calls pedestrian (14 for VOC, 0 for COCO)")
    ap.add_argument("--benchmark", choices=sorted(MOT_BENCHMARKS), default="MOT17")
    ap.add_argument("--obj_thresh", type=float, default=0.5)
    ap.add_argument("--iou_thresh", type=float, default=0.5, help="NMS IoU threshold")
    ap.add_argument("--max_per_class", type=int, default=100)
    add_track_args(ap)
    ap.add_argument("--streams", type=streams_arg, default=1, metavar="N",
                    help="track up to N sequences at once, in the same batches, each its own stream (the results do not "
                         "depend on N; each stream holds the tracker's state on the device)")
    ap.add_argument("--results", default=None, metavar="DIR", help="write DIR/<name>.txt in MOTChallenge tracker format")
    ap.add_argument("--out", default=None, help="write the table as JSON")
    return ap


def main():
    args = build_parser().parse_args()
    res = evaluate(args)
    if res is None:
        return
    print(report(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(to_json(res), fh)


if __name__ == "__main__":
    main()
