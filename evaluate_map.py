#!/usr/bin/env python
"""A checkpoint's mAP on an annotated image list (the .npy make_voc_list.py writes), with the matching, the per-class
ranking and the AP reduction on the GPU (evaluate.DetectionAP).

    python evaluate_map.py CKPT ANN.npy [--model_def yolo_mobilev1 --depth_multiplier 0.75 --image_size 224 320 --class_num 20
                                         --anchors data/voc_anchor.npy --batch 32 --obj_thresh 0.01 --iou_thresh 0.5
                                         --max_per_class 30 --eval_iou 0.5 0.55 ... 0.95 --out map.json]
    python -m torch.distributed.run --nproc-per-node 8 evaluate_map.py ...   # one rank per GPU; rank 0 evaluates

The files go through serve.py's batching loop (DetectionPipeline.submit_images: baseline JPEGs are decoded on the GPU, two
batches in flight), and rank 0 feeds every gathered record block to the evaluator.  Protocol (oracle/ap_ref.py): VOC
matching at each --eval_iou threshold (the first also gives the VOC 2007 11-point AP), IoU without a "+1 pixel" term, and
every object counts (the lists carry no "difficult" flag).  The defaults report AP at 0.5 and the mean over 0.50:0.05:0.95.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from serve import ModelArgParser, add_model_args, detect_files, load_image, open_pipeline  # noqa: E402
from k210_yolo_framework_b200.evaluate import DetectionAP, load_voc_annotations  # noqa: E402
from k210_yolo_framework_b200.preprocess import inspect_jpeg, inspect_png  # noqa: E402

COCO_IOU = [round(0.5 + 0.05 * i, 2) for i in range(10)]


def load_checked(path, hw, gpu_png=False, gpu_progressive=False):
    """load_image, refusing a file whose size differs from its annotation row's (the boxes would land elsewhere).  The size of
    a file kept compressed comes from its header (JPEG, progressive JPEG with `gpu_progressive`, or PNG with `gpu_png`)."""
    img = load_image(path, gpu_png, gpu_progressive) if gpu_png or gpu_progressive else load_image(path)
    if isinstance(img, (bytes, bytearray, memoryview)):
        got = tuple((inspect_png if bytes(img[:4]) == b"\x89PNG" else inspect_jpeg)(img)[:2])
    else:
        got = tuple(img.shape[:2])
    if got != tuple(hw):
        raise ValueError(f"{path}: decoded size {got[0]}x{got[1]} differs from its annotation's {hw[0]}x{hw[1]}")
    return img


def evaluate(args):
    """The result dict of DetectionAP on rank 0 (None on the other ranks)."""
    import torch.distributed as dist
    paths, labels, hw = load_voc_annotations(args.ann)
    pipe, world, rank = open_pipeline(args, args.max_per_class)
    ev = DetectionAP(args.class_num, args.max_per_class, args.eval_iou, device=pipe.device_index) if rank == 0 else None
    idx = list(range(len(paths)))
    gpu_png, gpu_progressive = getattr(args, "gpu_png", False), getattr(args, "gpu_progressive", False)
    for chunk, dets, counts in detect_files(pipe, idx, args.decode_threads, lambda i: load_checked(paths[i], hw[i], gpu_png, gpu_progressive)):
        if ev is not None:
            ev.update(dets[:len(chunk)], counts[:len(chunk)], [(labels[i], hw[i]) for i in chunk])
    if world > 1:
        dist.barrier()
    return ev.result() if ev is not None else None


def report(res, thresholds, names=None):
    """The per-class table (AP at each threshold, the 11-point AP at the first) and the means, as text."""
    C = len(res["npos"])
    names = names or [str(c) for c in range(C)]
    head = ["class", "npos", f"AP07@{thresholds[0]:g}"] + [f"AP@{t:g}" for t in thresholds]
    rows = [[names[c], str(int(res["npos"][c])), f"{res['ap07'][c]:.4f}"] + [f"{res['ap'][t, c]:.4f}" for t in range(len(thresholds))]
            for c in range(C)]
    rows.append(["mAP", str(int(res["npos"].sum())), f"{res['map07']:.4f}"] + [f"{m:.4f}" for m in res["map"]])
    width = [max(len(r[i]) for r in rows + [head]) for i in range(len(head))]
    lines = ["  ".join(v.rjust(w) for v, w in zip(r, width)) for r in [head] + rows]
    if len(thresholds) > 1:
        lines.append(f"mAP averaged over IoU {', '.join(f'{t:g}' for t in thresholds)}: {float(np.mean(res['map'])):.4f}")
    return "\n".join(lines)


def to_json(res, thresholds):
    out = {"iou_thresholds": list(thresholds), "map_mean": float(np.mean(res["map"]))}
    for k, v in res.items():
        out[k] = np.asarray(v).tolist() if not isinstance(v, float) else v
    return out


def main():
    ap = ModelArgParser()
    add_model_args(ap)
    ap.add_argument("ann", help="annotation list (.npy of (path, labels [n, 5] (class, x, y, w, h) relative, (h, w)) rows)")
    ap.add_argument("--obj_thresh", type=float, default=0.01)
    ap.add_argument("--iou_thresh", type=float, default=0.5, help="NMS IoU threshold")
    ap.add_argument("--max_per_class", type=int, default=30)
    ap.add_argument("--eval_iou", type=float, nargs="+", default=COCO_IOU,
                    help="matching IoU thresholds (1 to 16); the 11-point AP is reported at the first")
    ap.add_argument("--out", default=None, help="write the result dict as JSON")
    args = ap.parse_args()
    res = evaluate(args)
    if res is None:
        return
    print(report(res, args.eval_iou))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(to_json(res, args.eval_iou), fh)


if __name__ == "__main__":
    main()
