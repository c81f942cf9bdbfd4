"""MotEval on the GPU equals oracle/mot_ref.py exactly (counts, MOTP_sum, the ratios and the CLEAR rounds) on seeded
sequences, ties, empty frames, distractors, a long chain of ambiguous frames and several sequences at once, from device or
pinned host blocks; its refusals; and evaluate_mot.py end to end against mot_ref and sort_ref."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from mot_sequences import blocks, sequence
from oracle import mot_ref, sort_ref
from test_mot_ref import _chain

pytestmark = pytest.mark.gpu
PERSON = 14


def _frames_of(trk, L):
    """Tracker rows [n, 7] as the frames' records (id, (ymin, xmin, ymax, xmax), score), boxes exact in float32."""
    out = [[] for _ in range(L)]
    for f, t, left, top, w, h, s in trk.tolist():
        out[int(f) - 1].append((int(t), (top - 1, left - 1, top - 1 + h, left - 1 + w), s))
    return out


def _run(benchmark, seqs, device_views=True, split=37, seed=0):
    """MotEval's result over seqs [(name, gt, frames, L)], frames fed in shuffled batches of `split`; and mot_ref's."""
    from k210_yolo_framework_b200.evaluate import MotEval
    rng = np.random.default_rng(seed)
    ev = MotEval(benchmark, device=0)
    ref = {}
    for name, gt, frames, L in seqs:
        ev.add_sequence(name, gt, L)
    for name, gt, frames, L in seqs:
        ids, boxes, dets, counts = blocks(frames, rng=rng)
        trk = mot_ref.tracker_rows(range(L), ids, boxes, dets, counts, PERSON)
        ref[name] = mot_ref.evaluate(name, gt, trk, L, benchmark, by_rounds=True)
        assert {k: v for k, v in ref[name].items() if k != "rounds"} == mot_ref.evaluate(name, gt, trk, L, benchmark)
        starts = list(range(0, L, split))
        rng.shuffle(starts)
        for a in starts:
            sl = slice(a, a + split)
            blk = [torch.from_numpy(np.ascontiguousarray(x[sl])) for x in (ids, boxes, dets, counts)]
            blk = [b.cuda() for b in blk] if device_views else [b.pin_memory() for b in blk]
            ev.update(name, range(a, min(a + split, L)), *blk, PERSON)
    return ev.result(), ref


def _check(res, ref):
    for name, r in ref.items():
        r = dict(r)
        assert res["rounds"][name] == r.pop("rounds"), name
        assert res["sequences"][name] == r, name
    assert res["combined"] == mot_ref.combine(list(ref.values()))


@pytest.mark.parametrize("benchmark,L,n_ped,seed", [("MOT17", 200, 21, 0), ("MOT20", 150, 40, 1), ("MOT15", 120, 15, 2),
                                                    ("MOT17", 1050, 45, 3)])
def test_equals_mot_ref_on_seeded_sequences(benchmark, L, n_ped, seed):
    gt, frames = sequence(np.random.default_rng(seed), L, n_ped=n_ped, ambiguous=0.4, benchmark=benchmark)
    res, ref = _run(benchmark, [("s", gt, frames, L)], seed=seed)
    _check(res, ref)
    assert ref["s"]["IDSW"] > 0 and res["solved"]["s"] > 0


def test_several_sequences_ties_chains_empty_frames_and_an_empty_tracker_from_host_blocks():
    seqs = []
    for k in range(3):
        gt, frames = sequence(np.random.default_rng(20 + k), 90, ambiguous=0.5)
        for f in range(10 + k, 20 + k):
            frames[f] = []                       # frames without tracker rows
        seqs.append((f"seq{k}", gt[gt[:, 0] % 17 != 0], frames, 90))     # and frames without gt rows
    gt, trk = _chain(60)
    seqs.append(("chain", gt, _frames_of(trk, 60), 60))
    dup = [[(t, b, s), (t + 100, b, s)] for f in _frames_of(trk, 60) for (t, b, s) in f[:1]]     # duplicate boxes
    seqs.append(("dup", gt, dup, 60))
    seqs.append(("empty", gt, [[] for _ in range(60)], 60))
    for device_views in (False, True):
        res, ref = _run("MOT17", seqs, device_views=device_views, split=8)
        _check(res, ref)
    assert res["rounds"]["chain"] > 20
    assert res["sequences"]["empty"]["FN"] == len(gt) and res["sequences"]["empty"]["IDF1"] == 0.0


def test_calls_on_different_streams_stay_ordered():
    """Updates on a side stream held back by a sleeping kernel, result() on the default stream: the same numbers."""
    from k210_yolo_framework_b200.evaluate import MotEval
    gt, frames = sequence(np.random.default_rng(7), 60, ambiguous=0.4)
    ids, boxes, dets, counts = (torch.from_numpy(x).cuda() for x in blocks(frames))
    ref = mot_ref.evaluate("s", gt, mot_ref.tracker_rows(range(60), *(t.cpu() for t in (ids, boxes, dets, counts)), PERSON), 60)
    ev = MotEval("MOT17", device=0)
    ev.add_sequence("s", gt, 60)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        ev.update("s", range(60), ids, boxes, dets, counts, PERSON)
    res = ev.result()
    assert res["sequences"]["s"] == ref
    assert ev.result()["sequences"]["s"] == ref      # a second result() gives the same


def test_refusals():
    from k210_yolo_framework_b200.evaluate import MotEval
    gt, frames = sequence(np.random.default_rng(1), 20)
    ids, boxes, dets, counts = (torch.from_numpy(x) for x in blocks(frames))
    ev = MotEval("MOT17", device=0)
    with pytest.raises(ValueError, match="outside 1..13"):
        ev.add_sequence("bad", np.array([[1, 1, 0, 0, 5, 5, 1, 14.0]]), 20)
    crowd = np.array([[1, i, 0, 0, 5, 5, 1, 1.0] for i in range(513)])
    with pytest.raises(ValueError, match="more than 512"):
        ev.add_sequence("crowd", crowd, 20)
    ev.add_sequence("s", gt, 20)
    with pytest.raises(ValueError, match="frame position 20 is outside"):
        ev.update("s", [20], ids[:1], boxes[:1], dets[:1], counts[:1], PERSON)
    ev.update("s", [0], ids[:1], boxes[:1], dets[:1], counts[:1], PERSON)
    with pytest.raises(ValueError, match="frame 1 was given twice"):
        ev.update("s", [0], ids[:1], boxes[:1], dets[:1], counts[:1], PERSON)
    ev.result()
    for what, edit in (("appears twice", lambda i, b: i[0, PERSON, :2].fill_(77)),
                       ("2\\^22", lambda i, b: i.__setitem__((0, PERSON, 0), 1 << 22)),
                       ("not finite", lambda i, b: b.__setitem__((0, PERSON, 0, 2), float("inf")))):
        i2, b2 = ids[1:2].clone(), boxes[1:2].clone()
        edit(i2, b2)
        ev2 = MotEval("MOT17", device=0)
        ev2.add_sequence("s", gt, 20)
        ev2.update("s", [1], i2, b2, dets[1:2], counts[1:2], PERSON)
        with pytest.raises(ValueError, match=what):
            ev2.result()


# ---------------------------------------------------------------------------------------------------------------------
# evaluate_mot.py
# ---------------------------------------------------------------------------------------------------------------------
def _mot_sequence(tmp_path, name="PEOPLE-01", L=9, gt=True):
    """A sequence of people.jpg shifted a few pixels per frame (JPEG files), its gt the shifted golden people boxes."""
    from PIL import Image
    src = Image.open(os.path.join(GOLDEN, "people.jpg")).convert("RGB")
    W, H = src.size
    d = tmp_path / name
    (d / "img1").mkdir(parents=True)
    for k in range(L):
        canvas = Image.new("RGB", (W, H), (90, 90, 90))
        canvas.paste(src, (4 * k - 12, 2 * k - 6))
        canvas.save(d / "img1" / f"{k + 1:06d}.jpg", quality=92)
    (d / "seqinfo.ini").write_text(f"[Sequence]\nname={name}\nimDir=img1\nframeRate=30\nseqLength={L}\nimWidth={W}\n"
                                   f"imHeight={H}\nimExt=.jpg\n")
    if gt:
        (d / "gt").mkdir()
        rows = []
        for k in range(L):
            for i, (x, y, w, h) in enumerate([(60, 40, 80, 200), (200, 50, 70, 180), (330, 60, 60, 170)]):
                rows.append(f"{k + 1},{i + 1},{x + 4 * k - 12},{y + 2 * k - 6},{w},{h},1,1,1")
        (d / "gt" / "gt.txt").write_text("\n".join(rows) + "\n")
    return d


def _args(tmp_path, seqs, **kw):
    import evaluate_mot
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    from k210_yolo_framework_b200.yolonet import load_npz_weights
    ckpt = tmp_path / "model.h5"
    if not ckpt.exists():
        save_keras_weights(str(ckpt), load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    argv = [str(ckpt)] + [str(s) for s in seqs] + ["--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "4",
                                                   "--obj_thresh", "0.3", "--person_class", str(PERSON), "--track_min_hits", "1"]
    for k, v in kw.items():
        argv += [f"--{k}", str(v)]
    return evaluate_mot.build_parser().parse_args(argv)


def _read_results(path):
    rows = np.loadtxt(path, delimiter=",", dtype=np.float64, ndmin=2)
    return rows[:, :7].reshape(-1, 7)


def _sort_rows(args, d, L):
    """sort_ref over the untracked records of the sequence's frames, as tracker rows."""
    import serve
    from evaluate_map import load_checked
    from k210_yolo_framework_b200.evaluate import read_seqinfo
    info = read_seqinfo(str(d))
    files = [os.path.join(d, "img1", f"{k + 1:06d}.jpg") for k in range(L)]
    pipe, _, _ = serve.open_pipeline(args, args.max_per_class)
    C, K = args.class_num, args.max_per_class
    s = sort_ref.Sort(C, K, args.track_max_age, args.track_min_hits, args.track_iou)
    rows = []
    for chunk, dets, counts in serve.detect_files(pipe, list(range(L)), 2,
                                                  lambda k: load_checked(files[k], (info["imHeight"], info["imWidth"]))):
        for j, k in enumerate(chunk):
            d_ = dets[j].numpy()
            ids, bx = s.update(k, d_[..., :4].copy().view(np.float32), counts[j].numpy())
            rows.append(mot_ref.tracker_rows([k], ids[None], bx[None], d_[None], counts[j].numpy()[None], PERSON))
    return np.concatenate(rows)


def test_evaluate_mot_end_to_end(tmp_path):
    import evaluate_mot
    d1 = _mot_sequence(tmp_path / "train", "PEOPLE-01", 9)
    d2 = _mot_sequence(tmp_path / "train", "PEOPLE-02", 6)
    d3 = _mot_sequence(tmp_path / "test", "PEOPLE-03", 5, gt=False)
    out = tmp_path / "res"
    args = _args(tmp_path, [tmp_path / "train", d3], results=out)
    res = evaluate_mot.evaluate(args)
    assert set(res["sequences"]) == {"PEOPLE-01", "PEOPLE-02"}
    refs = []
    for d, name, L in ((d1, "PEOPLE-01", 9), (d2, "PEOPLE-02", 6)):
        trk = _read_results(out / f"{name}.txt")
        assert len(trk) > 5
        assert np.array_equal(trk, _sort_rows(args, d, L))
        gt = np.loadtxt(d / "gt" / "gt.txt", delimiter=",", ndmin=2)[:, :8]
        refs.append(mot_ref.evaluate(name, gt, trk, L))
        assert res["sequences"][name] == refs[-1]
    assert res["combined"] == mot_ref.combine(refs)
    assert os.path.isfile(out / "PEOPLE-03.txt")
    # the results as the gt: perfect
    trk = _read_results(out / "PEOPLE-01.txt")
    (d1 / "gt" / "gt.txt").write_text("".join(f"{int(r[0])},{int(r[1])},{r[2]!r},{r[3]!r},{r[4]!r},{r[5]!r},1,1,1\n"
                                              for r in trk.tolist()))
    res = evaluate_mot.evaluate(_args(tmp_path, [d1]))
    p = res["sequences"]["PEOPLE-01"]
    assert p["MOTA"] == p["IDF1"] == p["MOTP"] == 1.0
    text = evaluate_mot.report(res)
    assert "COMBINED" in text and "IDF1" in text


def test_evaluate_mot_refuses_missing_frames_and_nothing_to_do(tmp_path):
    import evaluate_mot
    d = _mot_sequence(tmp_path, "PEOPLE-01", 4)
    os.remove(d / "img1" / "000003.jpg")
    with pytest.raises(ValueError, match="000003.jpg is missing"):
        evaluate_mot.evaluate(_args(tmp_path, [d]))
    e = _mot_sequence(tmp_path, "PEOPLE-02", 3, gt=False)
    with pytest.raises(ValueError, match="nothing to do"):
        evaluate_mot.evaluate(_args(tmp_path, [e]))
    f = _mot_sequence(tmp_path, "PEOPLE-03", 3)
    (f / "seqinfo.ini").write_text((f / "seqinfo.ini").read_text().replace("imWidth=", "imWidth=1"))
    with pytest.raises(ValueError, match="differs"):
        evaluate_mot.evaluate(_args(tmp_path, [f]))


def test_two_gpus_give_the_single_gpu_numbers(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import json
    import evaluate_mot
    d = _mot_sequence(tmp_path, "PEOPLE-01", 11)
    args = _args(tmp_path, [d])
    one = evaluate_mot.to_json(evaluate_mot.evaluate(args))
    argv = [args.ckpt, str(d), "--anchors", args.anchors, "--batch", "4", "--obj_thresh", "0.3", "--person_class", str(PERSON),
            "--track_min_hits", "1", "--out", str(tmp_path / "two.json")]
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29561", os.path.join(ROOT, "evaluate_mot.py")] + argv,
                       capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert json.load(open(tmp_path / "two.json")) == json.loads(json.dumps(one))
