#!/usr/bin/env python
"""Times DetectionAP (k2y_ap_match per update + k2y_ap_result) against the numpy protocol (oracle/ap_ref.py) on seeded
synthetic record blocks at VOC07-test size (4952 images, C = 20, K = 30) and COCO-val size (5000 images, C = 80, K = 100),
1 to 10 ground-truth boxes per image, scores on a 0.01 grid so that many tie across images, and checks that both give the
same npos and TP flags and APs within 1e-9.  Prints the card's name, power limit and SM clock, read in the same run.

    python scripts/bench_eval.py [--batch 32] [--warmup 1] [--skip_oracle]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DET_DTYPE = np.dtype([("ymin", "<f4"), ("xmin", "<f4"), ("ymax", "<f4"), ("xmax", "<f4"), ("score", "<f4"), ("index", "<i4")])
THRESHOLDS = [round(0.5 + 0.05 * i, 2) for i in range(10)]


def synthetic_batch(seed, n, C, K, mean_dets=8.0, gt_range=(1, 10), empty_every=0):
    """One seeded batch: (dets int32 [n, C, K, 6], counts int32 [n, C], gt [(labels [g, 5] relative, (h, w))] * n).
    Detections of a class are jittered copies of its ground-truth boxes or random boxes, in score-descending record order;
    some (image, class) pairs have none; scores lie on a 0.01 grid, so many tie.  Every `empty_every`-th image has no
    ground truth (0: none)."""
    rng = np.random.default_rng(seed)
    rec = np.zeros((n, C, K), DET_DTYPE)
    counts = np.minimum(rng.geometric(1.0 / (1.0 + mean_dets), (n, C)) - 1, K).astype(np.int32)
    counts[rng.random((n, C)) < 0.3] = 0
    gt = []
    for b in range(n):
        H, W = (int(v) for v in rng.integers(120, 640, 2))
        g = 0 if empty_every and b % empty_every == empty_every - 1 else int(rng.integers(gt_range[0], gt_range[1] + 1))
        cls = rng.integers(0, C, g)
        xy = rng.random((g, 2)) * 0.8 + 0.1
        wh = rng.random((g, 2)) * 0.4 + 0.02
        labels = np.concatenate([cls[:, None], xy, wh], 1)
        gt.append((labels, (H, W)))
        boxes = np.stack([(xy[:, 1] - wh[:, 1] / 2) * H, (xy[:, 0] - wh[:, 0] / 2) * W, (xy[:, 1] + wh[:, 1] / 2) * H,
                          (xy[:, 0] + wh[:, 0] / 2) * W], 1)
        for c in np.nonzero(counts[b])[0]:
            m = int(counts[b, c])
            mine = boxes[cls == c]
            out = rng.random((m, 4)) * [H, W, H, W]
            out[:, 2:] = out[:, :2] + rng.random((m, 2)) * [H / 3, W / 3]
            if len(mine):
                pick = rng.random(m) < 0.6
                src = mine[rng.integers(0, len(mine), m)]
                jit = src + rng.normal(0, 0.08, (m, 4)) * np.repeat(src[:, 2:] - src[:, :2], 2, 1)
                out[pick] = jit[pick]
            score = np.sort(np.round(rng.random(m), 2))[::-1].astype(np.float32)
            r = rec[b, c, :m]
            r["ymin"], r["xmin"], r["ymax"], r["xmax"] = (out[:, i].astype(np.float32) for i in range(4))
            r["score"], r["index"] = score, np.arange(m)
    return rec.view(np.int32).reshape(n, C, K, 6), counts, gt


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(name, n_images, C, K, mean_dets, batch, warmup, oracle):
    import torch
    from k210_yolo_framework_b200.evaluate import DetectionAP
    dev = torch.device("cuda", 0)
    batches = []
    for s, b0 in enumerate(range(0, n_images, batch)):
        d, c, g = synthetic_batch(1000 + s, min(batch, n_images - b0), C, K, mean_dets)
        batches.append((torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev), g))
    n_rec = sum(int(c.sum()) for _, c, _ in batches)
    ev = DetectionAP(C, K, THRESHOLDS, device=0)
    for _ in range(warmup):
        for d, c, g in batches:
            ev.update(d, c, g)
        ev.result()
        ev.reset()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h0 = time.perf_counter()
    t0.record()
    for d, c, g in batches:
        ev.update(d, c, g)
    t1.record()
    res = ev.result()
    h1 = time.perf_counter()
    t1.synchronize()
    upd_ms = t0.elapsed_time(t1)
    print(f"{name}: {n_images} images, C={C}, K={K}, T={len(THRESHOLDS)}, {n_rec} records, {len(batches)} updates of {batch}")
    print(f"  GPU: update x{len(batches)} + result {1e3 * (h1 - h0):.1f} ms wall (updates {upd_ms:.1f} ms device time, "
          f"including the host's ground-truth packing), mAP@0.5 {res['map'][0]:.4f}, mAP@0.5:0.95 {np.mean(res['map']):.4f}")
    if not oracle:
        return
    from oracle.ap_ref import ApRef
    ref = ApRef(C, K, THRESHOLDS)
    h0 = time.perf_counter()
    for d, c, g in batches:
        ref.update(d.cpu().numpy(), c.cpu().numpy(), g)
    want = ref.result()
    h1 = time.perf_counter()
    print(f"  numpy oracle: {h1 - h0:.2f} s")
    flags = ev.tp_flags()
    assert np.array_equal(res["npos"], want["npos"]), "npos differs"
    assert np.array_equal(flags, np.stack(ref.tp_flags)), "TP flags differ"
    for k in ("ap", "ap07", "map"):
        a, b = np.asarray(res[k]), np.asarray(want[k])
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.nanmax(np.abs(a - b)) <= 1e-9, f"{k} differs"
    print(f"  identical npos and TP flags; max |AP - oracle| = {np.nanmax(np.abs(res['ap'] - want['ap'])):.2e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip_oracle", action="store_true")
    args = ap.parse_args()
    print("card (name, power limit, SM clock, max SM clock):", card_info())
    run("VOC07-test", 4952, 20, 30, 8.0, args.batch, args.warmup, not args.skip_oracle)
    run("COCO-val", 5000, 80, 100, 12.0, args.batch, args.warmup, not args.skip_oracle)
    print("card after the run:", card_info())


if __name__ == "__main__":
    main()
