"""ByteTrack on the GPU: ``k2y_bytetrack_update`` equals oracle/bytetrack_ref.py bit for bit (ids and float32 boxes) on seeded
record streams, whatever the batches they are split into; ``serve.py --track --tracker bytetrack`` keeps the untracked lines
records and adds the ids the oracle gives on them; ``evaluate_mot.py --tracker bytetrack`` scores the oracle's tracks; two
GPUs write what one writes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bytetrack_streams import crowded, stream
from conftest import ROOT
from oracle import bytetrack_ref
from test_gpu_track import WORKER, _equal

pytestmark = pytest.mark.gpu


def _block(frames, C, K, dev):
    """The frames as a gather block (records with their scores, then counts per row), frame i in row 2 i + 1."""
    from k210_yolo_framework_b200.dist import DetectionGather
    n = 2 * len(frames) + 1
    buf = torch.zeros((n, C * (K * 6 + 1)), dtype=torch.int32)
    dets, counts = DetectionGather.split(buf, C, K)
    for i, (b, c, s) in enumerate(frames):
        dets[2 * i + 1, :, :, :4] = torch.from_numpy(b.view(np.int32))
        dets[2 * i + 1, :, :, 4] = torch.from_numpy(s.view(np.int32))
        counts[2 * i + 1] = torch.from_numpy(c)
    return DetectionGather.split(buf.to(dev), C, K)


def _run(tracker, frames, positions, split, C, K, dev):
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
    t = bytetrack_ref.ByteTrack(C, K, **kw)
    out = [t.update(p, *f) for p, f in zip(positions, frames)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


@pytest.mark.parametrize("seed,C,K,kw", [
    (0, 20, 30, {}), (1, 20, 30, dict(track_buffer=0)), (2, 20, 30, dict(track_buffer=1, fuse_score=False)),
    (3, 80, 100, {}), (4, 80, 100, dict(track_buffer=1, fuse_score=False, track_thresh=0.6, match_thresh=0.9))])
def test_kernel_equals_bytetrack_ref_in_any_split(seed, C, K, kw):
    from k210_yolo_framework_b200.track import ByteTracker
    dev = torch.device("cuda", 0)
    frames = stream(np.random.default_rng(seed), C, K, 60, n_obj=40 if K == 100 else 12,
                    track_thresh=kw.get("track_thresh", 0.5))
    positions = list(range(60))
    ref = _ref(frames, positions, C, K, **kw)
    assert (ref[0] >= 0).sum() > 100
    for split in (1, 7, 32):
        t = ByteTracker(C, K, device=0, **kw)
        _equal(*_run(t, frames, positions, split, C, K, dev), *ref, f"split {split}")


def test_a_crowded_class_equals_the_oracle():
    from k210_yolo_framework_b200.track import ByteTracker
    C, K, B = 80, 100, 38        # 4000 tracks per class, the largest setting at K = 100
    frames = crowded(C, K, 2 * B + 6)
    positions = list(range(len(frames)))
    t_ref = bytetrack_ref.ByteTrack(C, K, track_buffer=B)
    ref, live = [], 0
    for p, f in zip(positions, frames):
        ref.append(t_ref.update(p, *f))
        live = max(live, len(t_ref.tracked[0]) + len(t_ref.lost[0]))
    assert live >= K * (B // 2 + 1)
    t = ByteTracker(C, K, track_buffer=B, device=0)
    _equal(*_run(t, frames, positions, 16, C, K, torch.device("cuda", 0)), np.stack([r[0] for r in ref]),
           np.stack([r[1] for r in ref]), "crowded")


def test_gaps_reset_and_refused_positions():
    from k210_yolo_framework_b200.track import ByteTracker
    C, K = 4, 30
    dev = torch.device("cuda", 0)
    frames = stream(np.random.default_rng(7), C, K, 40)
    positions = [p + (3 if p > 10 else 0) + (40 if p > 30 else 0) for p in range(40)]     # gaps of 4 and of 41
    positions[5:] = [p + 1 for p in positions[5:]]                                       # and one of 2
    kw = dict(track_buffer=3)
    ref = _ref(frames, positions, C, K, **kw)
    t = ByteTracker(C, K, device=0, **kw)
    _equal(*_run(t, frames, positions, 6, C, K, dev), *ref, "gaps")
    with pytest.raises(ValueError):
        t.check_positions([positions[-1]])
    t.reset()
    again = [p - 5 for p in range(5, 45)]
    _equal(*_run(t, frames, again, 9, C, K, dev), *_ref(frames, again, C, K, **kw), "after reset")


# ---------------------------------------------------------------------------------------------------------------------
# serve.py --track --tracker bytetrack
# ---------------------------------------------------------------------------------------------------------------------
def _track_ref(lines, C=20, K=30, **kw):
    """bytetrack_ref over the records of serve.py's lines: (ids, boxes) per detection, in line order."""
    t = bytetrack_ref.ByteTrack(C, K, **kw)
    out = []
    for line in lines:
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        where = []
        for d in line["detections"]:
            c = d["class"]
            boxes[c, counts[c]] = d["box_tlbr"]
            scores[c, counts[c]] = d["score"]
            where.append((c, counts[c]))
            counts[c] += 1
        ids, bx = t.update(line["frame"], boxes, counts, scores)
        out.append([(int(ids[c, k]), bx[c, k].tolist()) for c, k in where])
    return out


def _args01(tmp_path, p, batch, **kw):
    from test_gpu_video import _args
    a = _args(tmp_path, p, batch, **kw)
    a.obj_thresh = 0.1
    return a


@pytest.mark.parametrize("kw,batch", [({}, 4), ({"tiles": (1, 2), "flip": True}, 12)])
def test_serve_bytetrack_adds_the_oracle_ids_to_the_untracked_records(tmp_path, kw, batch):
    from test_gpu_video import _mjpeg_video, _serve
    p, _ = _mjpeg_video(tmp_path, 15)
    n0, plain = _serve(_args01(tmp_path, p, batch, **kw))
    a = _args01(tmp_path, p, batch, track=True, **kw)
    a.tracker = "bytetrack"
    n, tracked = _serve(a)
    assert n == n0 == 15
    plain, tracked = [json.loads(l) for l in plain], [json.loads(l) for l in tracked]
    for x, y in zip(plain, tracked):
        assert {k: v for k, v in x.items() if k != "detections"} == {k: v for k, v in y.items() if k != "detections"}
        assert [{k: v for k, v in d.items() if not k.startswith("track")} for d in y["detections"]] == x["detections"]
    ref = _track_ref(plain)
    got = [[(d["track"] if d["track"] is not None else -1, d.get("track_box_tlbr", [0.0] * 4)) for d in l["detections"]]
           for l in tracked]
    assert got == ref
    assert sum(t >= 0 for line in ref for t, _ in line) > 5


def test_two_gpus_track_what_one_tracks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_video import _mjpeg_video, _serve
    p, _ = _mjpeg_video(tmp_path, 13)
    a = _args01(tmp_path, p, 4, track=True, tiles=(1, 1))
    a.tracker = "bytetrack"
    n, one = _serve(a)
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    argv = [a.ckpt, str(p), "--anchors", a.anchors, "--batch", "4", "--obj_thresh", "0.1", "--track", "--tracker", "bytetrack",
            "--tiles", "1", "1"]
    env = dict(os.environ, K2Y_ROOT=ROOT, PYTHONPATH=ROOT, K2Y_OUT=str(tmp_path / "two.jsonl"))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29548", str(script)] + argv, capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert open(tmp_path / "two.jsonl").read().splitlines() == one


# ---------------------------------------------------------------------------------------------------------------------
# evaluate_mot.py --tracker bytetrack
# ---------------------------------------------------------------------------------------------------------------------
def _mot_args(tmp_path, seqs, **kw):
    import evaluate_mot
    from test_gpu_mot import GOLDEN, PERSON, _args
    _args(tmp_path, seqs)           # writes the checkpoint
    argv = [str(tmp_path / "model.h5")] + [str(s) for s in seqs] + [
        "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "4", "--obj_thresh", "0.1", "--person_class",
        str(PERSON), "--tracker", "bytetrack"]
    for k, v in kw.items():
        argv += [f"--{k}"] + ([] if v is True else [str(v)])
    return evaluate_mot.build_parser().parse_args(argv)


def _bytetrack_rows(args, d, L):
    """bytetrack_ref over the untracked records of the sequence's frames, as tracker rows."""
    import serve
    from evaluate_map import load_checked
    from k210_yolo_framework_b200.evaluate import read_seqinfo
    from oracle import mot_ref
    from test_gpu_mot import PERSON
    info = read_seqinfo(str(d))
    files = [os.path.join(d, "img1", f"{k + 1:06d}.jpg") for k in range(L)]
    pipe, _, _ = serve.open_pipeline(args, args.max_per_class)
    C, K = args.class_num, args.max_per_class
    t = bytetrack_ref.ByteTrack(C, K, args.track_thresh, args.track_match, args.track_buffer, not args.track_no_fuse_score)
    rows = []
    for chunk, dets, counts in serve.detect_files(pipe, list(range(L)), 2,
                                                  lambda k: load_checked(files[k], (info["imHeight"], info["imWidth"]))):
        for j, k in enumerate(chunk):
            d_ = dets[j].numpy()
            ids, bx = t.update(k, d_[..., :4].copy().view(np.float32), counts[j].numpy(), d_[..., 4].copy().view(np.float32))
            rows.append(mot_ref.tracker_rows([k], ids[None], bx[None], d_[None], counts[j].numpy()[None], PERSON))
    return np.concatenate(rows)


@pytest.mark.parametrize("kw", [{}, {"track_buffer": 2, "track_no_fuse_score": True}])
def test_evaluate_mot_bytetrack_equals_the_oracle_tracks(tmp_path, kw):
    import evaluate_mot
    from oracle import mot_ref
    from test_gpu_mot import _mot_sequence, _read_results
    d1 = _mot_sequence(tmp_path / "train", "PEOPLE-01", 9)
    d2 = _mot_sequence(tmp_path / "train", "PEOPLE-02", 6)
    out = tmp_path / "res"
    args = _mot_args(tmp_path, [tmp_path / "train"], results=out, **kw)
    res = evaluate_mot.evaluate(args)
    assert set(res["sequences"]) == {"PEOPLE-01", "PEOPLE-02"}
    refs = []
    for d, name, L in ((d1, "PEOPLE-01", 9), (d2, "PEOPLE-02", 6)):
        trk = _read_results(out / f"{name}.txt")
        assert len(trk) > 5
        assert np.array_equal(trk, _bytetrack_rows(args, d, L))
        gt = np.loadtxt(d / "gt" / "gt.txt", delimiter=",", ndmin=2)[:, :8]
        refs.append(mot_ref.evaluate(name, gt, trk, L))
        assert res["sequences"][name] == refs[-1]
    assert res["combined"] == mot_ref.combine(refs)
