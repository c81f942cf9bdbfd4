#!/usr/bin/env python
"""Tracking evaluation on the GPU (evaluate.MotEval: CLEAR, Identity and HOTA) against the host (oracle/mot_ref.py,
oracle/mot_hota_ref.py and their literal numpy / scipy forms)
on seeded synthetic data shaped like MOT17 train: 7 sequences of 600, 1050, 837, 525, 654, 900 and 750 frames, about 21
pedestrian gt rows per frame plus zero-marked and distractor rows, and tracker records made from the gt with jitter, misses,
false positives, ghost boxes, id switches and crossing pairs (tests/mot_sequences.py).

    python scripts/bench_mot_eval.py [--repeat 3] [--host 1]

It also times one denser sequence shaped like the crowded MOT20 train sequences on the GPU alone (600 frames, about 210 gt
rows and 200 tracker records per frame, about 900 pedestrian ids and 12.7 k tracker ids), where the identity assignment
is largest; the host forms are not run there (the literal form's square matrix alone would take 2.9 GB).

Prints the GPU evaluation time (create, every update from device blocks and result(), on a host clock around a device
synchronise, median of --repeat), the CLEAR rounds, the assignments solved over all rounds and the share of frames whose positives are not isolated
(the frames that need an assignment), the host times of
mot_ref and of the literal form, and of the HOTA restatement and its literal form (the results asserted identical to the
GPU's), the kernel time of the HOTA kernels and of the CLEAR and Identity kernels in a separate torch.profiler run of each
data set, and the card name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from mot_sequences import MOT17_TRAIN_LENGTHS, blocks, sequence  # noqa: E402
from k210_yolo_framework_b200.evaluate import MotEval  # noqa: E402

PERSON = 14


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        q = "unknown"
    return q


def gpu_eval(data, dev_blocks, benchmark="MOT17"):
    torch.cuda.synchronize()
    t = time.perf_counter()
    ev = MotEval(benchmark, device=0)
    for name, gt, L, blk in data:
        ev.add_sequence(name, gt, L)
    for name, gt, L, blk in data:
        for a in range(0, L, 32):
            ev.update(name, range(a, min(a + 32, L)), *(b[a:a + 32] for b in dev_blocks[name]), PERSON)
    res = ev.result()
    torch.cuda.synchronize()
    return time.perf_counter() - t, res


def kernel_shares(data, dev_blocks, benchmark="MOT17"):
    """One evaluation under torch.profiler: kernel time (ms) of the HOTA kernels, of the other evaluation kernels (CLEAR and
    Identity) and of all kernels."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gpu_eval(data, dev_blocks, benchmark)
    hota = other = 0.0
    per = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "hota_" in e.key:
            hota += t
            name = e.key[e.key.index("hota_"):].split("(")[0].split("<")[0].split("ENS")[0]
            per[name] = per.get(name, 0.0) + t / 1e3
        elif "mot_" in e.key:
            other += t
    return {"hota_kernels_ms": hota / 1e3, "clear_identity_kernels_ms": other / 1e3,
            "hota_by_kernel_ms": dict(sorted(per.items(), key=lambda kv: -kv[1]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--host", type=int, default=1, help="also time mot_ref and its literal form (0: no)")
    args = ap.parse_args()
    rng = np.random.default_rng(2017)
    data, dev_blocks = [], {}
    for i, L in enumerate(MOT17_TRAIN_LENGTHS):
        gt, frames = sequence(rng, L, n_ped=21, n_other=6, ambiguous=0.3)
        blk = blocks(frames, rng=rng)
        name = f"SYN17-{i:02d}"
        data.append((name, gt, L, blk))
        dev_blocks[name] = [torch.from_numpy(b).cuda() for b in (blk[0], blk[1], blk[2], blk[3])]
    gpu_eval(data, dev_blocks)          # warm-up: module load, allocations
    times, res = [], None
    for _ in range(args.repeat):
        t, res = gpu_eval(data, dev_blocks)
        times.append(t)
    n_frames = sum(L for _, _, L, _ in data)
    solved = sum(res["solved"].values())      # over every round
    out = {"card": card(), "sequences": len(data), "frames": n_frames,
           "gt_rows": int(sum(len(gt) for _, gt, _, _ in data)), "tracker_rows": res["combined"]["tracker_rows"],
           "gpu_s_median": float(np.median(times)), "gpu_s_all": times, "rounds": res["rounds"],
           "assignment_solves_all_rounds": solved,
           "MOTA": res["combined"]["MOTA"], "IDF1": res["combined"]["IDF1"]}
    if args.host:
        from oracle import mot_ref
        rows = {name: mot_ref.tracker_rows(range(L), *blk[:3], blk[3], PERSON) for name, gt, L, blk in data}
        t = time.perf_counter()
        ref = {name: mot_ref.evaluate(name, gt, rows[name], L) for name, gt, L, _ in data}
        out["mot_ref_s"] = time.perf_counter() - t
        t = time.perf_counter()
        lit = {name: mot_ref.evaluate_literal(gt, rows[name], L) for name, gt, L, _ in data}
        out["literal_s"] = time.perf_counter() - t
        fr = [f for name, gt, L, _ in data for f in mot_ref.preprocess(gt, rows[name], L)]
        hard = sum(1 for f in fr if f.gids and f.tids and not mot_ref.isolated(mot_ref.clear_score(f, {})))
        out["share_of_frames_needing_assignment"] = hard / n_frames
        for name in ref:
            assert ref[name] == lit[name] == res["sequences"][name], name
        assert mot_ref.combine(list(ref.values())) == res["combined"]
        from oracle import mot_hota_ref
        t = time.perf_counter()
        href = {name: mot_hota_ref.evaluate_hota(name, gt, rows[name], L) for name, gt, L, _ in data}
        out["hota_ref_s"] = time.perf_counter() - t
        t = time.perf_counter()
        hlit = {name: mot_hota_ref.evaluate_hota_literal(gt, rows[name], L) for name, gt, L, _ in data}
        out["hota_literal_s"] = time.perf_counter() - t
        for name in href:
            assert href[name] == hlit[name] == res["hota"]["sequences"][name], name
        assert mot_hota_ref.combine_hota(list(href.values())) == res["hota"]["combined"]
        out["identical"] = True
    out["HOTA"] = float(np.mean(res["hota"]["combined"]["HOTA"]))
    out["profile"] = kernel_shares(data, dev_blocks)
    gt, frames = sequence(np.random.default_rng(2020), 600, n_ped=1000, n_other=60, ambiguous=0.3, benchmark="MOT20",
                          life=(60, 180))
    blk = blocks(frames, K=320, rng=rng)
    dense = [("SYN20-00", gt, 600, blk)]
    dense_dev = {"SYN20-00": [torch.from_numpy(b).cuda() for b in blk]}
    gpu_eval(dense, dense_dev, "MOT20")
    times = []
    for _ in range(args.repeat):
        t, r20 = gpu_eval(dense, dense_dev, "MOT20")
        times.append(t)
    c = r20["combined"]
    out["mot20_shaped"] = {"frames": 600, "gt_rows": int(len(gt)), "max_gt_rows_per_frame": int(np.bincount(gt[:, 0].astype(int)).max()),
                           "tracker_rows": c["tracker_rows"], "gt_ids": len(np.unique(gt[(gt[:, 6] != 0) & (gt[:, 7] == 1), 1])),
                           "tracker_ids": len({t for f in frames for t, _, _ in f}), "gpu_s_median": float(np.median(times)),
                           "gpu_s_all": times, "rounds": r20["rounds"]["SYN20-00"], "MOTA": c["MOTA"], "IDF1": c["IDF1"],
                           "HOTA": float(np.mean(r20["hota"]["combined"]["HOTA"])),
                           "profile": kernel_shares(dense, dense_dev, "MOT20")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
