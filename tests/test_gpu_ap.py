"""DetectionAP (csrc/evaluate.cu) against the numpy protocol (oracle/ap_ref.py): seeded datasets over several updates,
device and pinned host record views, invalid records, evaluate_map.py end to end, and two GPUs."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle.ap_ref import ApRef

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_eval import synthetic_batch  # noqa: E402

pytestmark = pytest.mark.gpu


def thresholds(T):
    return [0.5] if T == 1 else [round(0.5 + 0.05 * i, 2) for i in range(T)]


def check_equal(ev, ref, res=None):
    res = ev.result() if res is None else res
    want = ref.result()
    assert np.array_equal(res["npos"], want["npos"])
    assert np.array_equal(ev.tp_flags(), np.stack(ref.tp_flags))
    for k in ("ap", "ap07", "map"):
        a, b = np.asarray(res[k], np.float64), np.asarray(want[k], np.float64)
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        assert np.nan_to_num(np.abs(a - b)).max() <= 1e-9, (k, a, b)
    assert (np.isnan(res["map07"]) and np.isnan(want["map07"])) or abs(res["map07"] - want["map07"]) <= 1e-9
    return res


@pytest.mark.parametrize("C,K,T", [(1, 1, 1), (1, 100, 10), (20, 30, 1), (20, 30, 10), (20, 1, 10), (80, 100, 1), (80, 30, 10)])
def test_matches_oracle_over_several_updates(C, K, T):
    from k210_yolo_framework_b200.evaluate import DetectionAP
    ev = DetectionAP(C, K, thresholds(T))
    ref = ApRef(C, K, thresholds(T))
    for s, n in enumerate([7, 1, 32, 20]):            # the store grows across updates
        d, c, g = synthetic_batch(100 * C + 10 * K + T + s, n, C, K, mean_dets=min(K, 6), empty_every=5)
        c[0] = 0                                       # an image without records
        ev.update(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), g)
        ref.update(d, c, g)
    check_equal(ev, ref)
    ev.reset()
    ref.reset()
    d, c, g = synthetic_batch(5, 9, C, K, mean_dets=min(K, 3))
    ev.update(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), g)
    ref.update(d, c, g)
    check_equal(ev, ref)


def test_single_class_above_2_pow_17_records_spans_many_ctas():
    from k210_yolo_framework_b200.evaluate import DetectionAP
    C, K = 2, 100
    ev, ref = DetectionAP(C, K, thresholds(10)), ApRef(C, K, thresholds(10))
    total = 0
    for s in range(14):
        d, c, g = synthetic_batch(7000 + s, 100, C, K, mean_dets=4)
        rec = d.view(np.dtype([("b", "<f4", 4), ("score", "<f4"), ("index", "<i4")]))[..., 0]
        c[:, 0] = K                                    # class 0 full in every image: 140,000 records
        empty = rec["score"][:, 0] == 0
        rec["b"][:, 0][empty] = [10, 10, 60, 60]
        rec["score"][:, 0][empty] = 0.25               # a large block of equal scores across images
        total += int(c[:, 0].sum())
        ev.update(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), g)
        ref.update(d, c, g)
    assert total > 2 ** 17
    check_equal(ev, ref)


def test_device_and_pinned_host_views_agree():
    """Records as a gather block: per-image records and counts adjacent (DetectionGather's layout), once as the device view
    step_device returns and once as the pinned host view collect returns."""
    from k210_yolo_framework_b200.dist import DetectionGather
    from k210_yolo_framework_b200.evaluate import DetectionAP
    C, K, n = 20, 30, 16
    evs = [DetectionAP(C, K, thresholds(10)) for _ in range(2)]
    ref = ApRef(C, K, thresholds(10))
    for s in range(3):
        d, c, g = synthetic_batch(300 + s, n, C, K, mean_dets=5)
        buf = np.zeros((n, C * (K * 6 + 1)), np.int32)
        buf[:, :C * K * 6] = d.reshape(n, -1)
        buf[:, C * K * 6:] = c
        host = torch.from_numpy(buf).pin_memory()
        dev = host.cuda()
        dd, dc = DetectionGather.split(dev, C, K)
        hd, hc = DetectionGather.split(host, C, K)
        evs[0].update(dd, dc, g)
        evs[1].update(hd, hc, g)
        host.zero_()                       # the host view may be overwritten once update returned
        ref.update(d, c, g)
    r0 = check_equal(evs[0], ref)
    r1 = evs[1].result()
    assert np.array_equal(evs[0].tp_flags(), evs[1].tp_flags())
    assert np.array_equal(r0["ap"], r1["ap"], equal_nan=True) and np.array_equal(r0["ap07"], r1["ap07"], equal_nan=True)


@pytest.mark.parametrize("bad", ["nan", "negative", "count"])
def test_invalid_records_make_result_raise(bad):
    from k210_yolo_framework_b200.evaluate import DetectionAP
    C, K = 4, 5
    d, c, g = synthetic_batch(9, 3, C, K, mean_dets=3)
    c[1, 2] = max(int(c[1, 2]), 1)
    rec = d.view(np.float32)
    if bad == "nan":
        rec[1, 2, 0, 4] = np.nan
    elif bad == "negative":
        rec[1, 2, 0, 4] = -0.5
    else:
        c[1, 2] = K + 1
    ev = DetectionAP(C, K)
    ev.update(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), g)
    with pytest.raises(ValueError, match="score" if bad != "count" else "count"):
        ev.result()
    ev.reset()
    d2, c2, g2 = synthetic_batch(10, 3, C, K, mean_dets=3)
    ev.update(torch.from_numpy(d2).cuda(), torch.from_numpy(c2).cuda(), g2)
    ev.result()                            # reset clears the status


def _args(ckpt, **kw):
    class A:
        pass
    a = A()
    a.ckpt, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.01, 0.5, 2
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _dataset(tmp_path, golden_weights):
    """dog.jpg / people.jpg and copies as JPEG files, labelled with the network's own confident boxes (some shifted)."""
    from PIL import Image
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    names = []
    for i in range(7):
        src = "dog.jpg" if i % 2 == 0 else "people.jpg"
        names.append(str(d / f"{i:02d}_{src}"))
        shutil.copy(os.path.join(GOLDEN, src), names[-1])
    with open(tmp_path / "conf.jsonl", "w") as fh:
        serve.serve(_args(ckpt, images=str(d), obj_thresh=0.7), fh)
    lines = [json.loads(l) for l in open(tmp_path / "conf.jsonl")]
    rows = np.empty((len(names), 3), object)
    for i, (name, line) in enumerate(zip(names, lines)):
        assert line["image"] == name
        H, W = Image.open(name).size[::-1]
        lab = []
        for k, det in enumerate(line["detections"]):
            y0, x0, y1, x1 = det["box_tlbr"]
            shift = 0.15 * (x1 - x0) * ((i + k) % 3)          # some boxes moved by 0, 15 or 30 % of their width
            lab.append([det["class"], ((x0 + x1) / 2 + shift) / W, (y0 + y1) / 2 / H, (x1 - x0) / W, (y1 - y0) / H])
        if i == 5:
            lab.append([3, 0.5, 0.5, 0.2, 0.2])               # an object nobody detects
        rows[i] = [name, np.array(lab, np.float64).reshape(-1, 5), np.array([H, W])]
    np.save(tmp_path / "ann.npy", rows)
    return ckpt, d, str(tmp_path / "ann.npy"), rows


def test_evaluate_map_end_to_end_matches_oracle_on_serve_output(tmp_path, golden_weights):
    import evaluate_map
    import serve
    ckpt, d, ann, rows = _dataset(tmp_path, golden_weights)
    thr = [0.5, 0.75, 0.9]
    res = evaluate_map.evaluate(_args(ckpt, ann=ann, max_per_class=30, eval_iou=thr))
    with open(tmp_path / "dets.jsonl", "w") as fh:
        serve.serve(_args(ckpt, images=str(d)), fh)
    C, K = 20, 30
    ref = ApRef(C, K, thr)
    for row, line in zip(rows, (json.loads(l) for l in open(tmp_path / "dets.jsonl"))):
        rec = np.zeros((1, C, K), np.dtype([("b", "<f4", 4), ("score", "<f4"), ("index", "<i4")]))
        cnt = np.zeros((1, C), np.int32)
        for det in line["detections"]:
            c = det["class"]
            rec[0, c, cnt[0, c]] = (det["box_tlbr"], det["score"], det["index"])
            cnt[0, c] += 1
        ref.update(rec.view(np.int32).reshape(1, C, K, 6), cnt, [(row[1], row[2])])
    want = ref.result()
    assert np.array_equal(res["npos"], want["npos"]) and res["npos"].sum() > 0
    for k in ("ap", "ap07", "map"):
        assert np.allclose(res[k], want[k], atol=1e-9, rtol=0, equal_nan=True), k
    assert 0 < res["map"][0] < 1
    text = evaluate_map.report(res, thr)
    assert "mAP" in text and len(text.splitlines()) == C + 3      # header, C classes, the means, the mean over thresholds


def test_evaluate_map_rejects_a_size_mismatch(tmp_path, golden_weights):
    import evaluate_map
    ckpt, d, ann, rows = _dataset(tmp_path, golden_weights)
    rows[4][2] = np.array([rows[4][2][0] + 1, rows[4][2][1]])
    np.save(tmp_path / "bad.npy", rows)
    with pytest.raises(ValueError, match="04_dog.jpg"):
        evaluate_map.evaluate(_args(ckpt, ann=str(tmp_path / "bad.npy"), max_per_class=30, eval_iou=[0.5]))


def test_two_gpus_give_the_single_gpu_result(tmp_path, golden_weights):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ckpt, d, ann, rows = _dataset(tmp_path, golden_weights)
    outs = []
    for world in (1, 2):
        out = tmp_path / f"map{world}.json"
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
               "127.0.0.1", "--master-port", str(29620 + world), os.path.join(ROOT, "evaluate_map.py"), str(ckpt), ann,
               "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "2", "--out", str(out)]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(json.load(open(out)))
    assert sorted(outs[0]) == sorted(outs[1])
    for k in outs[0]:
        assert np.array_equal(np.asarray(outs[0][k], np.float64), np.asarray(outs[1][k], np.float64), equal_nan=True), k
