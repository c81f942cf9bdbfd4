#!/usr/bin/env python
"""A checkpoint's COCO numbers on a COCO instances file: the 12 lines pycocotools' COCOeval(gt, dt, "bbox").summarize()
prints and the AP of every category, with the matching, ranking and curves on the GPU (evaluate.CocoEval).

    python evaluate_coco.py CKPT instances_val2017.json IMAGE_DIR [--model_def yolo --class_num 80 --image_size 416 416
                                                                    --anchors ANCHORS.npy --batch 32 --obj_thresh 0.001
                                                                    --iou_thresh 0.5 --max_per_class 100
                                                                    --results dets.json --out coco.json]
    python -m torch.distributed.run --nproc-per-node 8 evaluate_coco.py ...   # one rank per GPU; rank 0 evaluates

Every image the file lists is read from IMAGE_DIR/file_name, in sorted image-id order, through serve.py's batching loop;
a file whose size differs from the file's height / width raises ValueError.  Class index c of the network is the c-th
smallest category id (the order of Darknet's coco.names), so the file must list class_num categories.  --results writes
the detections as a COCO results file (what the COCO evaluation server takes); --out the stats and per-category AP.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from evaluate_map import load_checked  # noqa: E402
from serve import ModelArgParser, add_model_args, detect_files, open_pipeline  # noqa: E402
from k210_yolo_framework_b200.evaluate import CocoEval, coco_results, coco_summary, load_coco_annotations  # noqa: E402


def evaluate(args):
    """(result dict of CocoEval, category ids) on rank 0, (None, category ids) on the other ranks."""
    import torch.distributed as dist
    images, cats, gt = load_coco_annotations(args.ann)
    if len(cats) != args.class_num:
        raise ValueError(f"{args.ann} lists {len(cats)} categories, the network has {args.class_num} classes")
    pipe, world, rank = open_pipeline(args, args.max_per_class)
    ev = CocoEval(gt, args.class_num, args.max_per_class, device=pipe.device_index) if rank == 0 else None
    results = [] if rank == 0 and getattr(args, "results", None) else None
    paths = [os.path.join(args.image_dir, im[1]) for im in images]
    idx = list(range(len(images)))
    gpu_png, gpu_progressive = getattr(args, "gpu_png", False), getattr(args, "gpu_progressive", False)
    for chunk, dets, counts in detect_files(pipe, idx, args.decode_threads, lambda i: load_checked(paths[i], images[i][2], gpu_png, gpu_progressive)):
        if ev is None:
            continue
        ev.update(dets[:len(chunk)], counts[:len(chunk)], chunk)
        if results is not None:
            results += coco_results(dets[:len(chunk)], counts[:len(chunk)], [images[i][0] for i in chunk], cats)
    if world > 1:
        dist.barrier()
    if ev is None:
        return None, cats
    if results is not None:
        with open(args.results, "w") as fh:
            json.dump(results, fh)
    return ev.result(), cats


def report(res, cats, names=None):
    """The 12 summary lines, then AP (IoU 0.50:0.95, area all, maxDets 100) per category."""
    names = names or [str(c) for c in cats]
    lines = coco_summary(res["stats"])
    width = max(len(n) for n in names + ["category"])
    lines.append(f"{'category'.rjust(width)}  {'id':>4}  AP")
    for n, c, v in zip(names, cats, res["ap_per_class"]):
        lines.append(f"{n.rjust(width)}  {c:>4}  {v:.4f}")
    return "\n".join(lines)


def to_json(res, cats):
    return {"stats": [float(v) for v in res["stats"]], "category_ids": list(cats),
            "ap_per_class": [None if np.isnan(v) else float(v) for v in res["ap_per_class"]]}


def main():
    ap = ModelArgParser()
    add_model_args(ap)
    ap.add_argument("ann", help="COCO instances JSON file")
    ap.add_argument("image_dir", help="directory holding the listed file_name of every image")
    ap.add_argument("--obj_thresh", type=float, default=0.001)
    ap.add_argument("--iou_thresh", type=float, default=0.5, help="NMS IoU threshold")
    ap.add_argument("--max_per_class", type=int, default=100)
    ap.add_argument("--results", default=None, help="write the detections as a COCO results JSON file")
    ap.add_argument("--out", default=None, help="write the stats and per-category AP as JSON")
    args = ap.parse_args()
    res, cats = evaluate(args)
    if res is None:
        return
    print(report(res, cats))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(to_json(res, cats), fh)


if __name__ == "__main__":
    main()
