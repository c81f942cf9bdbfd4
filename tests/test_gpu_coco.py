"""CocoEval (csrc/evaluate.cu) against the Python restatement of COCOeval (oracle/coco_ref.py): seeded datasets over
several class counts and K, updates in shuffled image order, device and pinned host record views, invalid records and
positions, evaluate_coco.py end to end, and two GPUs."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle.coco_ref import DET_DTYPE, CocoRef, records_to_results

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_coco_eval import load, synthetic_coco  # noqa: E402

pytestmark = pytest.mark.gpu


def oracle(ds, dets, counts):
    ids = sorted(im["id"] for im in ds["images"])
    return CocoRef(ds).evaluate(records_to_results(dets, counts, ids, sorted(c["id"] for c in ds["categories"])))


def assert_equal(res, want):
    for k in ("precision", "recall", "stats"):
        assert np.array_equal(res[k], want[k]), (k, np.argwhere(res[k] != want[k])[:5])
    assert np.array_equal(res["ap_per_class"], want["ap_per_class"], equal_nan=True)


def run(gt, dets, counts, C, K, seed, splits=4, device_views=True):
    from k210_yolo_framework_b200.evaluate import CocoEval
    ev = CocoEval(gt, C, K)
    order = np.random.default_rng(seed).permutation(len(dets))
    for part in np.array_split(order, splits):
        d, c = torch.from_numpy(dets[part].copy()), torch.from_numpy(counts[part].copy())
        if device_views:
            d, c = d.cuda(), c.cuda()
        ev.update(d, c, part)
    return ev


@pytest.mark.parametrize("C,K,n", [(1, 1, 9), (1, 100, 12), (3, 10, 20), (20, 30, 24), (20, 100, 16), (80, 100, 12),
                                   (5, 150, 14), (7, 250, 6)])
def test_matches_oracle_in_shuffled_updates(C, K, n):
    ds, dets, counts = synthetic_coco(100 * C + K + n, n, C, K, mean_dets=min(K, 6), empty_every=5)
    counts[1] = 0                                          # an image without records
    if K > 100:
        counts[2, 0] = K                                   # more than COCOeval's 100 per (image, class)
        rec = dets.view(DET_DTYPE)[..., 0]
        rec[2, 0]["score"] = np.linspace(0.99, 0.0, K).round(2).astype(np.float32)
        rec[2, 0]["ymax"] = rec[2, 0]["ymin"] + 30
        rec[2, 0]["xmax"] = rec[2, 0]["xmin"] + 30
    ids = sorted(im["id"] for im in ds["images"])
    for a in ds["annotations"]:                            # image 3: all crowd
        if a["image_id"] == ids[3]:
            a["iscrowd"] = 1
    _, _, gt = load(ds)
    ev = run(gt, dets, counts, C, K, seed=n)
    want = oracle(ds, dets, counts)
    assert_equal(ev.result(), want)
    ev.reset()
    part = np.arange(0, n, 2)                              # after a reset: only half the images have records
    ev.update(torch.from_numpy(dets[part].copy()).cuda(), torch.from_numpy(counts[part].copy()).cuda(), part)
    c2 = np.zeros_like(counts)
    c2[part] = counts[part]
    assert_equal(ev.result(), oracle(ds, dets, c2))


def test_classes_without_ground_truth_and_boundary_areas():
    C, K, n = 10, 20, 10
    ds, dets, counts = synthetic_coco(77, n, C, K, mean_dets=4)
    cats = sorted(c["id"] for c in ds["categories"])
    ds["annotations"] = [a for a in ds["annotations"] if a["category_id"] not in cats[:3]]   # 3 classes without ground truth
    for i, a in enumerate(ds["annotations"]):
        a["area"] = [1024.0, 9216.0, a["area"]][i % 3]
    _, _, gt = load(ds)
    want = oracle(ds, dets, counts)
    assert np.isnan(want["ap_per_class"][:3]).all() and (want["precision"][:, :, :3] == -1).all()
    assert_equal(run(gt, dets, counts, C, K, seed=3).result(), want)


def test_device_and_pinned_host_views_agree():
    """Records as a gather block (per-image records and counts adjacent), once as the device view step_device returns
    and once as the pinned host view collect returns."""
    from k210_yolo_framework_b200.dist import DetectionGather
    from k210_yolo_framework_b200.evaluate import CocoEval
    C, K, n = 20, 30, 24
    ds, dets, counts = synthetic_coco(300, n, C, K, mean_dets=5)
    _, _, gt = load(ds)
    evs = [CocoEval(gt, C, K) for _ in range(2)]
    order = np.random.default_rng(1).permutation(n)
    for part in np.array_split(order, 3):
        m = len(part)
        buf = np.zeros((m, C * (K * 6 + 1)), np.int32)
        buf[:, :C * K * 6] = dets[part].reshape(m, -1)
        buf[:, C * K * 6:] = counts[part]
        host = torch.from_numpy(buf).pin_memory()
        dev = host.cuda()
        evs[0].update(*DetectionGather.split(dev, C, K), torch.from_numpy(part).cuda())
        evs[1].update(*DetectionGather.split(host, C, K), part)
        host.zero_()                       # the host view may be overwritten once update returned
    want = oracle(ds, dets, counts)
    assert_equal(evs[0].result(), want)
    assert_equal(evs[1].result(), want)


@pytest.mark.parametrize("bad,match", [("nan", "score"), ("negative", "score"), ("count", "count"),
                                       ("position", "position"), ("repeat", "twice"), ("repeat_later", "twice")])
def test_invalid_records_and_positions_make_result_raise(bad, match):
    from k210_yolo_framework_b200.evaluate import CocoEval
    C, K, n = 4, 5, 6
    ds, dets, counts = synthetic_coco(9, n, C, K, mean_dets=3)
    _, _, gt = load(ds)
    counts[1, 2] = max(int(counts[1, 2]), 1)
    pos = np.arange(n)
    rec = dets.view(np.float32)
    if bad == "nan":
        rec[1, 2, 0, 4] = np.nan
    elif bad == "negative":
        rec[1, 2, 0, 4] = -0.5
    elif bad == "count":
        counts[1, 2] = K + 1
    elif bad == "position":
        pos[4] = n
    elif bad == "repeat":
        pos[4] = 2
    ev = CocoEval(gt, C, K)
    ev.update(torch.from_numpy(dets).cuda(), torch.from_numpy(counts).cuda(), pos)
    if bad == "repeat_later":
        ev.update(torch.from_numpy(dets[:1]).cuda(), torch.from_numpy(counts[:1]).cuda(), [3])
    with pytest.raises(ValueError, match=match):
        ev.result()
    ev.reset()
    _, d2, c2 = synthetic_coco(9, n, C, K, mean_dets=3)
    ev.update(torch.from_numpy(d2).cuda(), torch.from_numpy(c2).cuda(), np.arange(n))
    assert_equal(ev.result(), oracle(ds, d2, c2))           # reset clears the status


def test_class_count_must_match_the_categories():
    from k210_yolo_framework_b200.evaluate import CocoEval
    ds, _, _ = synthetic_coco(5, 3, 4, 5)
    _, _, gt = load(ds)
    with pytest.raises(ValueError, match="categories"):
        CocoEval(gt, 5, 5)


def _args(ckpt, **kw):
    class A:
        pass
    a = A()
    a.ckpt, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.001, 0.5, 2
    a.max_per_class, a.results = 100, None
    for k, v in kw.items():
        setattr(a, k, v)
    return a


CATS = [2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61, 67, 71]


def _dataset(tmp_path, golden_weights):
    """dog.jpg / people.jpg copies and an instances file with 20 non-contiguous category ids, annotated with the network's
    own confident boxes (some shifted, one crowd, one object nobody detects, one image without annotations)."""
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
        names.append(f"{i:02d}_{src}")
        shutil.copy(os.path.join(GOLDEN, src), d / names[-1])
    with open(tmp_path / "conf.jsonl", "w") as fh:
        serve.serve(_args(ckpt, images=str(d), obj_thresh=0.7), fh)
    lines = [json.loads(l) for l in open(tmp_path / "conf.jsonl")]
    ids = [50 - 6 * i for i in range(7)]                   # sorted id order is the reverse of the file order
    images, anns = [], []
    for i, (name, line) in enumerate(zip(names, lines)):
        W, H = Image.open(d / name).size
        images.append({"id": ids[i], "file_name": name, "height": H, "width": W})
        if i == 3:
            continue
        for k, det in enumerate(line["detections"]):
            y0, x0, y1, x1 = det["box_tlbr"]
            shift = 0.15 * (x1 - x0) * ((i + k) % 3)
            anns.append({"image_id": ids[i], "category_id": CATS[det["class"]], "bbox": [x0 + shift, y0, x1 - x0, y1 - y0],
                         "area": (x1 - x0) * (y1 - y0) * 0.8, "iscrowd": int(i == 5 and k == 0)})
        if i == 5:
            anns.append({"image_id": ids[i], "category_id": CATS[3], "bbox": [100, 100, 40, 40], "area": 1600.0,
                         "iscrowd": 0})
    for j, a in enumerate(anns):
        a["id"] = 1000 + 7 * j
    ds = {"images": images, "annotations": anns, "categories": [{"id": c, "name": f"c{c}"} for c in CATS[::-1]]}
    (tmp_path / "inst.json").write_text(json.dumps(ds))
    return ckpt, d, str(tmp_path / "inst.json"), ds


def test_evaluate_coco_end_to_end_matches_oracle(tmp_path, golden_weights):
    import evaluate_coco
    from evaluate_map import load_checked
    from serve import detect_files, open_pipeline
    ckpt, d, ann, ds = _dataset(tmp_path, golden_weights)
    args = _args(ckpt, ann=ann, image_dir=str(d), results=str(tmp_path / "res.json"))
    res, cats = evaluate_coco.evaluate(args)
    assert cats == CATS
    # the oracle on the records the same pipeline gives for the same files (sorted image-id order), and on --results
    order = sorted(ds["images"], key=lambda im: im["id"])
    pipe, _, _ = open_pipeline(args, args.max_per_class)
    blocks = []
    for chunk, dets, counts in detect_files(pipe, list(range(len(order))), 2,
                                            lambda i: load_checked(str(d / order[i]["file_name"]), (order[i]["height"], order[i]["width"]))):
        blocks.append((dets[:len(chunk)].numpy().copy(), counts[:len(chunk)].numpy().copy()))
    dets, counts = (np.concatenate(x) for x in zip(*blocks))
    assert counts.sum() > 0
    want = oracle(ds, dets, counts)
    assert_equal(res, want)
    file_res = CocoRef(ds).evaluate(json.load(open(tmp_path / "res.json")))
    assert_equal(file_res, want)
    assert 0 < res["stats"][1] <= 1
    text = evaluate_coco.report(res, cats)
    assert len(text.splitlines()) == 12 + 1 + 20 and "Average Precision  (AP) @[ IoU=0.50:0.95" in text


def test_two_gpus_give_the_single_gpu_stats(tmp_path, golden_weights):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    ckpt, d, ann, ds = _dataset(tmp_path, golden_weights)
    outs = []
    for world in (1, 2):
        out = tmp_path / f"coco{world}.json"
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
               "127.0.0.1", "--master-port", str(29640 + world), os.path.join(ROOT, "evaluate_coco.py"), str(ckpt), ann, str(d),
               "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "2", "--out", str(out)]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(json.load(open(out)))
    assert outs[0] == outs[1]
