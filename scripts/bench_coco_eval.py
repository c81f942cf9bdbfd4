#!/usr/bin/env python
"""Times CocoEval (k2y_coco_match per update + k2y_coco_result) at COCO-val size on seeded synthetic data, and checks it
against the Python restatement of COCOeval (oracle/coco_ref.py) on the first --oracle_images images.

The data: 5000 images with ids listed out of order, C = 80 categories with non-contiguous ids, K = 100 records per
class; about 7 ground-truth boxes per image, about 1 % of them crowd, box sizes over the small / medium / large ranges
and some areas of exactly 1024 and 9216; records are jittered ground-truth boxes or random boxes with scores on a 0.01
grid (many tie across images).  Updates of 32 images arrive in shuffled image order.  Prints the card's name, power limit
and SM clock, read in the same run.

    python scripts/bench_coco_eval.py [--images 5000] [--batch 32] [--warmup 1] [--oracle_images 300]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_eval import DET_DTYPE, card_info  # noqa: E402


def synthetic_coco(seed, n_images, C, K, mean_gt=7.0, mean_dets=12.0, crowd=0.01, empty_every=0):
    """(dataset, dets int32 [n, C, K, 6], counts int32 [n, C]): a COCO instances dict and the record blocks of its images
    in sorted image-id order.  Every `empty_every`-th image (sorted order) has no annotations (0: none)."""
    rng = np.random.default_rng(seed)
    img_ids = np.sort(rng.choice(np.arange(1, 40 * n_images + 2), n_images, replace=False))
    cat_ids = np.sort(rng.choice(np.arange(1, 3 * C + 2), C, replace=False))
    images, anns = [], []
    rec = np.zeros((n_images, C, K), DET_DTYPE)
    counts = np.minimum(rng.geometric(1.0 / (1.0 + mean_dets), (n_images, C)) - 1, K).astype(np.int32)
    counts[rng.random((n_images, C)) < 0.5] = 0
    for b in range(n_images):
        H, W = (int(v) for v in rng.integers(200, 640, 2))
        images.append({"id": int(img_ids[b]), "file_name": f"{img_ids[b]:012d}.jpg", "height": H, "width": W})
        g = 0 if empty_every and b % empty_every == empty_every - 1 else int(rng.poisson(mean_gt))
        cls = rng.integers(0, C, g)
        side = np.exp(rng.uniform(np.log(4), np.log(300), (g, 2)))            # small, medium and large boxes
        wh = np.minimum(side, [W - 1, H - 1])
        xy = rng.random((g, 2)) * ([W, H] - wh)
        area = wh[:, 0] * wh[:, 1] * rng.uniform(0.5, 1.0, g)                 # a segment inside its box
        area[rng.random(g) < 0.05] = 1024.0
        area[rng.random(g) < 0.05] = 9216.0
        is_crowd = rng.random(g) < crowd
        for j in range(g):
            anns.append({"image_id": int(img_ids[b]), "category_id": int(cat_ids[cls[j]]), "iscrowd": int(is_crowd[j]),
                         "bbox": [float(xy[j, 0]), float(xy[j, 1]), float(wh[j, 0]), float(wh[j, 1])],
                         "area": float(area[j])})
        tlbr = np.stack([xy[:, 1], xy[:, 0], xy[:, 1] + wh[:, 1], xy[:, 0] + wh[:, 0]], 1)
        for c in np.nonzero(counts[b])[0]:
            m = int(counts[b, c])
            out = rng.random((m, 4)) * [H, W, H, W]
            out[:, 2:] = out[:, :2] + rng.random((m, 2)) * [H / 3, W / 3]
            mine = tlbr[cls == c]
            if len(mine):
                pick = rng.random(m) < 0.6
                src = mine[rng.integers(0, len(mine), m)]
                jit = src + rng.normal(0, 0.1, (m, 4)) * np.repeat(src[:, 2:] - src[:, :2], 2, 1)
                out[pick] = jit[pick]
            score = np.sort(np.round(rng.random(m), 2))[::-1].astype(np.float32)
            r = rec[b, c, :m]
            r["ymin"], r["xmin"], r["ymax"], r["xmax"] = (out[:, i].astype(np.float32) for i in range(4))
            r["score"], r["index"] = score, np.arange(m)
    ids = rng.permutation(np.arange(1, len(anns) + 1) * 3)                   # non-contiguous, in no particular order
    for a, i in zip(anns, ids):
        a["id"] = int(i)
    order = rng.permutation(len(anns))
    dataset = {"images": [images[i] for i in rng.permutation(n_images)], "annotations": [anns[i] for i in order],
               "categories": [{"id": int(c), "name": f"c{c}"} for c in rng.permutation(cat_ids)]}
    return dataset, rec.view(np.int32).reshape(n_images, C, K, 6), counts


def subset(dataset, n):
    """The dataset restricted to its first n images in sorted id order."""
    keep = set(sorted(im["id"] for im in dataset["images"])[:n])
    return {"images": [im for im in dataset["images"] if im["id"] in keep],
            "annotations": [a for a in dataset["annotations"] if a["image_id"] in keep], "categories": dataset["categories"]}


def load(dataset):
    from k210_yolo_framework_b200.evaluate import load_coco_annotations
    with tempfile.NamedTemporaryFile("w", suffix=".json", delete=False) as fh:
        json.dump(dataset, fh)
    try:
        return load_coco_annotations(fh.name)
    finally:
        os.unlink(fh.name)


def evaluate_gpu(gt, dets, counts, C, K, batch, seed, warmup=0):
    """(result, wall ms of the timed updates + result): updates of `batch` images in shuffled order."""
    import torch
    from k210_yolo_framework_b200.evaluate import CocoEval
    order = np.random.default_rng(seed).permutation(len(dets))
    d, c = torch.from_numpy(dets).cuda(), torch.from_numpy(counts).cuda()
    chunks = [torch.from_numpy(order[i:i + batch]).cuda() for i in range(0, len(order), batch)]
    parts = [(d[p].contiguous(), c[p].contiguous(), p) for p in chunks]
    ev = CocoEval(gt, C, K)
    for _ in range(warmup):
        for pd, pc, pp in parts:
            ev.update(pd, pc, pp)
        ev.result()
        ev.reset()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for pd, pc, pp in parts:
        ev.update(pd, pc, pp)
    res = ev.result()
    return res, 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--classes", type=int, default=80)
    ap.add_argument("--max_per_class", type=int, default=100)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--oracle_images", type=int, default=300, help="images of the oracle comparison (0: none)")
    args = ap.parse_args()
    C, K = args.classes, args.max_per_class
    print("card (name, power limit, SM clock, max SM clock):", card_info())
    dataset, dets, counts = synthetic_coco(2024, args.images, C, K)
    images, cats, gt = load(dataset)
    n_rec = int(np.minimum(counts, 100).sum())
    print(f"COCO-val size: {args.images} images, C={C}, K={K}, {len(gt.rows)} annotations "
          f"({int(gt.rows[:, 6].sum())} crowd), {n_rec} records evaluated, updates of {args.batch} in shuffled order")
    res, ms = evaluate_gpu(gt, dets, counts, C, K, args.batch, 7, args.warmup)
    print(f"  GPU: update x{-(-args.images // args.batch)} + result {ms:.1f} ms wall; AP {res['stats'][0]:.4f}, "
          f"AP50 {res['stats'][1]:.4f}, AR100 {res['stats'][8]:.4f}")
    if args.oracle_images:
        from oracle.coco_ref import CocoRef, records_to_results
        n = min(args.oracle_images, args.images)
        sub = subset(dataset, n)
        _, _, sub_gt = load(sub)
        got, _ = evaluate_gpu(sub_gt, dets[:n], counts[:n], C, K, args.batch, 8)
        t0 = time.perf_counter()
        want = CocoRef(sub).evaluate(records_to_results(dets[:n], counts[:n], [im[0] for im in images[:n]], cats))
        t1 = time.perf_counter()
        print(f"  oracle on the first {n} images: {t1 - t0:.2f} s")
        for k in ("precision", "recall", "stats"):
            assert np.array_equal(got[k], want[k]), f"{k} differs from the oracle"
        assert np.array_equal(got["ap_per_class"], want["ap_per_class"], equal_nan=True)
        print(f"  precision, recall, stats and per-class AP identical to the oracle (AP {want['stats'][0]:.4f})")
    print("card after the run:", card_info())


if __name__ == "__main__":
    main()
