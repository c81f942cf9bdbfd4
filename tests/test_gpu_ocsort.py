"""OC-SORT on the GPU: ``k2y_ocsort_update`` equals oracle/ocsort_ref.py bit for bit (ids and float32 boxes) on seeded record
streams, whatever the batches they are split into, on a class filled to its track bound, and across gaps, resets and refused
positions; ``serve.py --track --tracker ocsort`` keeps the untracked lines' records and adds the ids the oracle gives on them;
``evaluate_mot.py --tracker ocsort`` scores the oracle's tracks; two GPUs write what one writes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from ocsort_streams import crowded, stream
from oracle import ocsort_ref
from test_gpu_bytetrack import _run
from test_gpu_track import WORKER, _equal

pytestmark = pytest.mark.gpu


def _ref(frames, positions, C, K, **kw):
    t = ocsort_ref.OcSort(C, K, **kw)
    out = [t.update(p, *f) for p, f in zip(positions, frames)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


@pytest.mark.parametrize("seed,C,K,kw", [
    (0, 20, 30, {}), (1, 20, 30, dict(use_byte=True)), (2, 20, 30, dict(delta_t=1, max_age=5, min_hits=1)),
    (3, 80, 100, dict(max_age=9)), (4, 80, 100, dict(use_byte=True, delta_t=8, max_age=9, inertia=0.6, det_thresh=0.5))])
def test_kernel_equals_ocsort_ref_in_any_split(seed, C, K, kw):
    from k210_yolo_framework_b200.track import OcSortTracker
    dev = torch.device("cuda", 0)
    n = 60 if K == 30 else 30
    frames = stream(np.random.default_rng(seed), C, K, n, n_obj=40 if K == 100 else 12, max_age=kw.get("max_age", 30),
                    det_thresh=kw.get("det_thresh", 0.6))
    positions = list(range(n))
    ref = _ref(frames, positions, C, K, **kw)
    assert (ref[0] >= 0).sum() > 100
    for split in (1, 7, 32):
        t = OcSortTracker(C, K, device=0, **kw)
        _equal(*_run(t, frames, positions, split, C, K, dev), *ref, f"split {split}")


def test_a_class_filled_to_its_bound_equals_the_oracle():
    from k210_yolo_framework_b200.track import OcSortTracker
    C, K, A = 80, 30, 30            # 930 tracks in class 0, the default max_age at max_per_class 30
    frames = crowded(C, K, A + 6)
    positions = list(range(len(frames)))
    t_ref = ocsort_ref.OcSort(C, K, max_age=A)
    ref, live = [], 0
    for p, f in zip(positions, frames):
        ref.append(t_ref.update(p, *f))
        live = max(live, len(t_ref.tracks[0]))
    assert live == ocsort_ref.max_tracks(K, A)
    t = OcSortTracker(C, K, max_age=A, device=0)
    _equal(*_run(t, frames, positions, 16, C, K, torch.device("cuda", 0)), np.stack([r[0] for r in ref]),
           np.stack([r[1] for r in ref]), "filled")


def test_gaps_reset_and_refused_positions():
    from k210_yolo_framework_b200.track import OcSortTracker
    C, K = 4, 30
    dev = torch.device("cuda", 0)
    kw = dict(max_age=3, use_byte=True)
    frames = stream(np.random.default_rng(7), C, K, 40, max_age=3)
    positions = [p + (3 if p > 10 else 0) + (40 if p > 30 else 0) for p in range(40)]     # gaps of 4 and of 41
    positions[5:] = [p + 1 for p in positions[5:]]                                       # and one of 2
    ref = _ref(frames, positions, C, K, **kw)
    t = OcSortTracker(C, K, device=0, **kw)
    _equal(*_run(t, frames, positions, 6, C, K, dev), *ref, "gaps")
    with pytest.raises(ValueError):
        t.check_positions([positions[-1]])
    t.reset()
    again = [p - 5 for p in range(5, 45)]
    _equal(*_run(t, frames, again, 9, C, K, dev), *_ref(frames, again, C, K, **kw), "after reset")


# ---------------------------------------------------------------------------------------------------------------------
# serve.py --track --tracker ocsort
# ---------------------------------------------------------------------------------------------------------------------
def _track_ref(lines, C=20, K=30, **kw):
    """ocsort_ref over the records of serve.py's lines: (ids, boxes) per detection, in line order."""
    t = ocsort_ref.OcSort(C, K, **kw)
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


@pytest.mark.parametrize("kw,batch", [({}, 4), ({"tiles": (1, 2), "flip": True}, 12), ({"track_use_byte": True}, 4)])
def test_serve_ocsort_adds_the_oracle_ids_to_the_untracked_records(tmp_path, kw, batch):
    from test_gpu_video import _args, _mjpeg_video, _serve
    p, _ = _mjpeg_video(tmp_path, 15)
    view = {k: v for k, v in kw.items() if not k.startswith("track")}
    a0 = _args(tmp_path, p, batch, **view)
    a0.obj_thresh = 0.1
    n0, plain = _serve(a0)
    a = _args(tmp_path, p, batch, track=True, tracker="ocsort", **kw)
    a.obj_thresh = 0.1
    n, tracked = _serve(a)
    assert n == n0 == 15
    plain, tracked = [json.loads(l) for l in plain], [json.loads(l) for l in tracked]
    for x, y in zip(plain, tracked):
        assert {k: v for k, v in x.items() if k != "detections"} == {k: v for k, v in y.items() if k != "detections"}
        assert [{k: v for k, v in d.items() if not k.startswith("track")} for d in y["detections"]] == x["detections"]
    ref = _track_ref(plain, use_byte=bool(kw.get("track_use_byte")))
    got = [[(d["track"] if d["track"] is not None else -1, d.get("track_box_tlbr", [0.0] * 4)) for d in l["detections"]]
           for l in tracked]
    assert got == ref
    assert sum(t >= 0 for line in ref for t, _ in line) > 5


def test_two_gpus_track_what_one_tracks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_video import _args, _mjpeg_video, _serve
    p, _ = _mjpeg_video(tmp_path, 13)
    a = _args(tmp_path, p, 4, track=True, tracker="ocsort", tiles=(1, 1))
    n, one = _serve(a)
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    argv = [a.ckpt, str(p), "--anchors", a.anchors, "--batch", "4", "--obj_thresh", "0.3", "--track", "--tracker", "ocsort",
            "--tiles", "1", "1"]
    env = dict(os.environ, K2Y_ROOT=ROOT, PYTHONPATH=ROOT, K2Y_OUT=str(tmp_path / "two.jsonl"))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29549", str(script)] + argv, capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert open(tmp_path / "two.jsonl").read().splitlines() == one


# ---------------------------------------------------------------------------------------------------------------------
# evaluate_mot.py --tracker ocsort
# ---------------------------------------------------------------------------------------------------------------------
def _mot_args(tmp_path, seqs, **kw):
    import evaluate_mot
    from test_gpu_mot import GOLDEN, PERSON, _args
    _args(tmp_path, seqs)           # writes the checkpoint
    argv = [str(tmp_path / "model.h5")] + [str(s) for s in seqs] + [
        "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "4", "--obj_thresh", "0.1", "--person_class",
        str(PERSON), "--tracker", "ocsort"]
    for k, v in kw.items():
        argv += [f"--{k}"] + ([] if v is True else [str(v)])
    return evaluate_mot.build_parser().parse_args(argv)


def _ocsort_rows(args, d, L):
    """ocsort_ref over the untracked records of the sequence's frames, as tracker rows."""
    import serve
    from evaluate_map import load_checked
    from k210_yolo_framework_b200.evaluate import read_seqinfo
    from oracle import mot_ref
    from test_gpu_mot import PERSON
    info = read_seqinfo(str(d))
    files = [os.path.join(d, "img1", f"{k + 1:06d}.jpg") for k in range(L)]
    pipe, _, _ = serve.open_pipeline(args, args.max_per_class)
    C, K = args.class_num, args.max_per_class
    t = ocsort_ref.OcSort(C, K, args.track_det_thresh, args.track_max_age, args.track_min_hits, args.track_iou,
                          args.track_delta_t, args.track_inertia, args.track_use_byte)
    rows = []
    for chunk, dets, counts in serve.detect_files(pipe, list(range(L)), 2,
                                                  lambda k: load_checked(files[k], (info["imHeight"], info["imWidth"]))):
        for j, k in enumerate(chunk):
            d_ = dets[j].numpy()
            ids, bx = t.update(k, d_[..., :4].copy().view(np.float32), counts[j].numpy(), d_[..., 4].copy().view(np.float32))
            rows.append(mot_ref.tracker_rows([k], ids[None], bx[None], d_[None], counts[j].numpy()[None], PERSON))
    return np.concatenate(rows)


@pytest.mark.parametrize("kw", [{}, {"track_max_age": 2, "track_use_byte": True, "track_min_hits": 1}])
def test_evaluate_mot_ocsort_equals_the_oracle_tracks(tmp_path, kw):
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
        assert np.array_equal(trk, _ocsort_rows(args, d, L))
        gt = np.loadtxt(d / "gt" / "gt.txt", delimiter=",", ndmin=2)[:, :8]
        refs.append(mot_ref.evaluate(name, gt, trk, L))
        assert res["sequences"][name] == refs[-1]
    assert res["combined"] == mot_ref.combine(refs)
