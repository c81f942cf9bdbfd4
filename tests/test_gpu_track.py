"""SORT tracking on the GPU: ``k2y_track_update`` equals oracle/sort_ref.py bit for bit (ids and float32 boxes) on seeded record
streams, whatever the batches they are split into; ``serve.py --track`` keeps the untracked lines' records and adds the ids
sort_ref gives on them; two GPUs write what one writes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import sort_ref

pytestmark = pytest.mark.gpu


def _stream(rng, C, K, n_frames, n_obj=12, size=600.0):
    """[n_frames] of (boxes float32 [C, K, 4], counts [C]): per class objects that move, cross, hide and leave, records in random
    order with noise, identical duplicates (assignment ties), zero-area records and a few infinite boxes (NaN predictions)."""
    out = []
    objs = [[dict(start=int(rng.integers(0, n_frames)), life=int(rng.integers(2, n_frames)), p=rng.random(2) * size,
                  v=rng.normal(size=2) * 8, wh=8 + rng.random(2) * 70) for _ in range(int(rng.integers(0, n_obj)))] for _ in range(C)]
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        counts = np.zeros(C, np.int32)
        for c in range(C):
            recs = []
            for o in objs[c]:
                if o["start"] <= f < o["start"] + o["life"] and rng.random() < 0.85:
                    ctr = o["p"] + o["v"] * (f - o["start"]) + rng.normal(size=2) * 2
                    recs.append([ctr[1] - o["wh"][1] / 2, ctr[0] - o["wh"][0] / 2, ctr[1] + o["wh"][1] / 2, ctr[0] + o["wh"][0] / 2])
            if recs and rng.random() < 0.3:
                recs.append(list(recs[int(rng.integers(0, len(recs)))]))
            if rng.random() < 0.1:
                recs.append([3.0, 3.0, 3.0, 40.0])
            if rng.random() < 0.03:
                recs.append([0.0, 0.0, 10.0, np.inf])
            rng.shuffle(recs)
            recs = recs[:K]
            if recs:
                boxes[c, :len(recs)] = np.array(recs, np.float32)
            counts[c] = len(recs)
        out.append((boxes, counts))
    return out


def _crowded(C, K, n_frames):
    """Class 0 fills its track bound: K new boxes in each frame that overlap nothing, so every record is born (through an
    assignment of IoU 0 whose matches are all dropped) and K (max_age + 1) tracks are alive."""
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        for i in range(K):
            y, x = 20.0 * i, 100.0 + 20.0 * f
            boxes[0, i] = [y, x, y + 10, x + 10]
        counts = np.zeros(C, np.int32)
        counts[0] = K
        counts[C - 1] = 1
        boxes[C - 1, 0] = [5, 5, 50, 50 + f]
        out.append((boxes, counts))
    return out


def _block(frames, C, K, dev):
    """The frames as a gather block (records then counts per row), frame i in row 2 i + 1 (so the rows mapping is exercised)."""
    from k210_yolo_framework_b200.dist import DetectionGather
    n = 2 * len(frames) + 1
    buf = torch.zeros((n, C * (K * 6 + 1)), dtype=torch.int32)
    dets, counts = DetectionGather.split(buf, C, K)
    for i, (b, c) in enumerate(frames):
        dets[2 * i + 1, :, :, :4] = torch.from_numpy(b.view(np.int32))
        counts[2 * i + 1] = torch.from_numpy(c)
    return DetectionGather.split(buf.to(dev), C, K)


def _equal(ids, boxes, ref_ids, ref_boxes, what):
    assert np.array_equal(ids, ref_ids), what
    nan = np.isnan(ref_boxes)
    assert np.array_equal(np.isnan(boxes), nan), what
    assert np.array_equal(np.where(nan, 0, boxes).view(np.int32), np.where(nan, 0, ref_boxes).view(np.int32)), what


def _run(tracker, frames, positions, split, C, K, dev):
    """ids, boxes of the frames through `tracker`, in batches of `split` frames."""
    st = torch.cuda.current_stream()
    ids, boxes = [], []
    for a in range(0, len(frames), split):
        chunk, pos = frames[a:a + split], positions[a:a + split]
        dets, counts = _block(chunk, C, K, dev)
        rows = torch.tensor([2 * i + 1 for i in range(len(chunk))], dtype=torch.int32, device=dev)
        p = torch.tensor(tracker.check_positions(pos), dtype=torch.int64, device=dev)
        io_ = torch.full((len(chunk), C, K), 7, dtype=torch.int32, device=dev)
        bo = torch.full((len(chunk), C, K, 4), 7.0, dtype=torch.float32, device=dev)
        tracker.update(dets, counts, rows, p, len(chunk), io_, bo, st, pos[-1])
        ids.append(io_.cpu().numpy())
        boxes.append(bo.cpu().numpy())
    return np.concatenate(ids), np.concatenate(boxes)


def _ref(frames, positions, C, K, **kw):
    s = sort_ref.Sort(C, K, **kw)
    out = [s.update(p, b, c) for p, (b, c) in zip(positions, frames)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


@pytest.mark.parametrize("seed,C,K,max_age,min_hits,thresh", [
    (0, 20, 30, 1, 3, 0.3), (1, 20, 30, 4, 1, 0.3), (2, 20, 30, 0, 0, 0.1), (3, 80, 100, 9, 3, 0.3), (4, 3, 30, 33, 2, 0.5)])
def test_kernel_equals_sort_ref_in_any_split(seed, C, K, max_age, min_hits, thresh):
    from k210_yolo_framework_b200.track import Tracker
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(seed)
    frames = _stream(rng, C, K, 70, n_obj=40 if K == 100 else 12)
    positions = list(range(70))
    kw = dict(max_age=max_age, min_hits=min_hits, iou_thresh=thresh)
    ref = _ref(frames, positions, C, K, **kw)
    assert (ref[0] >= 0).sum() > 50
    for split in (1, 7, 32):
        t = Tracker(C, K, device=0, **kw)
        _equal(*_run(t, frames, positions, split, C, K, dev), *ref, f"split {split}")


def test_a_class_at_its_track_bound():
    from k210_yolo_framework_b200.track import Tracker
    C, K, max_age = 80, 100, 9
    frames = _crowded(C, K, 14)
    positions = list(range(14))
    s = sort_ref.Sort(C, K, max_age=max_age)
    ref = []
    for p, (b, c) in zip(positions, frames):
        ref.append(s.update(p, b, c))
        assert len(s.tracks[0]) <= 1000
    assert len(s.tracks[0]) == 1000
    t = Tracker(C, K, max_age=max_age, device=0)
    _equal(*_run(t, frames, positions, 7, C, K, torch.device("cuda", 0)), np.stack([r[0] for r in ref]),
           np.stack([r[1] for r in ref]), "crowded")


def test_gaps_and_reset():
    from k210_yolo_framework_b200.track import Tracker
    C, K = 4, 30
    dev = torch.device("cuda", 0)
    frames = _stream(np.random.default_rng(7), C, K, 40)
    positions = [p + (3 if p > 10 else 0) + (40 if p > 30 else 0) for p in range(40)]     # gaps of 4 and of 41
    positions[5:] = [p + 1 for p in positions[5:]]                                       # and one of 2
    kw = dict(max_age=3, min_hits=1)
    ref = _ref(frames, positions, C, K, **kw)
    t = Tracker(C, K, device=0, **kw)
    _equal(*_run(t, frames, positions, 6, C, K, dev), *ref, "gaps")
    with pytest.raises(ValueError):
        t.check_positions([positions[-1]])
    t.reset()
    again = [p - 5 for p in range(5, 45)]
    _equal(*_run(t, frames, again, 9, C, K, dev), *_ref(frames, again, C, K, **kw), "after reset")


# ---------------------------------------------------------------------------------------------------------------------
# serve.py --track
# ---------------------------------------------------------------------------------------------------------------------
def _track_ref(lines, C=20, K=30, **kw):
    """sort_ref over the records of serve.py's lines: (ids, boxes) per detection, in line order."""
    s = sort_ref.Sort(C, K, **kw)
    out = []
    for line in lines:
        boxes = np.zeros((C, K, 4), np.float32)
        counts = np.zeros(C, np.int32)
        where = []
        for d in line["detections"]:
            c = d["class"]
            boxes[c, counts[c]] = d["box_tlbr"]
            where.append((c, counts[c]))
            counts[c] += 1
        ids, bx = s.update(line["frame"], boxes, counts)
        out.append([(int(ids[c, k]), bx[c, k].tolist()) for c, k in where])
    return out


@pytest.mark.parametrize("kw,batch", [({}, 4), ({"tiles": (1, 2), "flip": True}, 12), ({}, 2)])
def test_serve_track_adds_sort_ids_to_the_untracked_records(tmp_path, kw, batch):
    from test_gpu_video import _args, _mjpeg_video, _serve
    p, stored = _mjpeg_video(tmp_path, 15)
    n0, plain = _serve(_args(tmp_path, p, batch, **kw))
    n, tracked = _serve(_args(tmp_path, p, batch, track=True, **kw))
    assert n == n0 == 15
    plain, tracked = [json.loads(l) for l in plain], [json.loads(l) for l in tracked]
    for a, b in zip(plain, tracked):
        assert {k: v for k, v in a.items() if k != "detections"} == {k: v for k, v in b.items() if k != "detections"}
        assert [{k: v for k, v in d.items() if not k.startswith("track")} for d in b["detections"]] == a["detections"]
    ref = _track_ref(plain)
    got = [[(d["track"] if d["track"] is not None else -1, d.get("track_box_tlbr", [0.0] * 4)) for d in l["detections"]]
           for l in tracked]
    assert got == ref
    assert sum(t >= 0 for line in ref for t, _ in line) > 5


WORKER = r'''
import io, os, sys
sys.path.insert(0, os.environ["K2Y_ROOT"])
import serve
args = serve.build_parser().parse_args(sys.argv[1:])
out = open(os.environ["K2Y_OUT"], "w") if int(os.environ["RANK"]) == 0 else None
serve.serve(args, out)
if out is not None:
    out.close()
'''


def test_two_gpus_track_what_one_tracks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_video import _args, _mjpeg_video, _serve
    p, _ = _mjpeg_video(tmp_path, 13)
    a = _args(tmp_path, p, 4, track=True, tiles=(1, 1))
    n, one = _serve(a)
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    argv = [a.ckpt, str(p), "--anchors", a.anchors, "--batch", "4", "--obj_thresh", "0.3", "--track", "--tiles", "1", "1"]
    env = dict(os.environ, K2Y_ROOT=ROOT, PYTHONPATH=ROOT, K2Y_OUT=str(tmp_path / "two.jsonl"))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29547", str(script)] + argv, capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert open(tmp_path / "two.jsonl").read().splitlines() == one
