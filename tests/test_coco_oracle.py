"""The COCO protocol (oracle/coco_ref.py) on hand-computed cases, the two-tier matching form, the instances loader's
refusals, the results-file round trip, the summary text, and (where pycocotools is installed) COCOeval itself."""
import json
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import coco_ref
from oracle.coco_ref import CocoRef, bb_iou, match_literal, match_two_tier, records_to_results

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_coco_eval import synthetic_coco  # noqa: E402

EPS = np.spacing(1)


def dataset(images, anns, cats=(1,)):
    """images: [(id, h, w)]; anns: [(image_id, category_id, bbox, area, iscrowd)], ids 1, 2, ... in list order."""
    return {"images": [{"id": i, "file_name": f"{i}.jpg", "height": h, "width": w} for i, h, w in images],
            "annotations": [{"id": k + 1, "image_id": i, "category_id": c, "bbox": list(b), "area": a, "iscrowd": z}
                            for k, (i, c, b, a, z) in enumerate(anns)],
            "categories": [{"id": c, "name": str(c)} for c in cats]}


def det(image_id, bbox, score, cat=1):
    return {"image_id": image_id, "category_id": cat, "bbox": list(bbox), "score": score}


def test_parameters_are_cocoevals_linspace_values():
    from k210_yolo_framework_b200.evaluate import COCO_IOU_THRS, COCO_REC_THRS
    assert COCO_IOU_THRS.tobytes() == np.linspace(.5, .95, 10).tobytes() == coco_ref.IOU_THRS.tobytes()
    assert COCO_REC_THRS.tobytes() == np.linspace(0, 1, 101).tobytes() == coco_ref.REC_THRS.tobytes()
    assert coco_ref.MAX_DETS == [1, 10, 100]
    assert coco_ref.AREA_RNG == [[0, 1e10], [0, 1024], [1024, 9216], [9216, 1e10]]
    assert np.where(.75 == COCO_IOU_THRS)[0].tolist() == [5] and np.where(.5 == COCO_IOU_THRS)[0].tolist() == [0]


def test_bbiou_uses_box_areas_and_the_detection_area_for_crowd():
    d, g = [[0.0, 0.0, 10.0, 10.0]], [[5.0, 5.0, 10.0, 10.0], [5.0, 5.0, 10.0, 10.0], [10.0, 0.0, 5.0, 5.0]]
    iou = bb_iou(d, g, [0, 1, 0])
    assert iou[0, 0] == 25.0 / 175.0           # i / (100 + 100 - 25)
    assert iou[0, 1] == 25.0 / 100.0           # crowd: i / area_d
    assert iou[0, 2] == 0.0                    # touching edges: iw = 0
    assert bb_iou([], g, [0, 0, 0]).shape == (0, 3)


def test_records_become_xywh_in_float64_of_the_float32_values():
    from k210_yolo_framework_b200.evaluate import coco_results
    rec = np.zeros((1, 2, 3), coco_ref.DET_DTYPE)
    rec[0, 1, 0] = (0.1, 0.7, 100.3, 50.9, 0.33, 4)
    rec[0, 1, 1] = (2.0, 3.0, 4.0, 5.0, 0.125, 5)
    dets, counts = rec.view(np.int32).reshape(1, 2, 3, 6), np.array([[0, 2]], np.int32)
    got = coco_results(dets, counts, [42], [3, 9])
    f = np.float32
    want = [{"image_id": 42, "category_id": 9, "score": float(f(0.33)),
             "bbox": [float(f(0.7)), float(f(0.1)), float(f(50.9)) - float(f(0.7)), float(f(100.3)) - float(f(0.1))]},
            {"image_id": 42, "category_id": 9, "bbox": [3.0, 2.0, 2.0, 2.0], "score": 0.125}]
    assert got == want == records_to_results(dets, counts, [42], [3, 9])


def test_one_tp_gives_precision_one_over_one_plus_eps():
    ev = CocoRef(dataset([(1, 100, 100)], [(1, 1, (10, 10, 20, 20), 400.0, 0)])).evaluate([det(1, (10, 10, 20, 20), 0.9)])
    p = ev["precision"]
    assert np.all(p[:, :, 0, 0, :] == 1.0 / (1.0 + EPS)) and 1.0 / (1.0 + EPS) < 1.0
    assert np.all(ev["recall"][:, 0, 0, :] == 1.0)
    assert np.all(p[:, :, 0, 1, :] == 1.0 / (1.0 + EPS))        # area 400: small
    assert np.all(p[:, :, 0, 2:, :] == -1) and np.all(ev["recall"][:, 0, 2:, :] == -1)   # no medium / large ground truth
    assert ev["stats"][0] == 1.0 / (1.0 + EPS) and ev["stats"][4] == -1


def test_area_bounds_belong_to_both_ranges_and_use_the_area_field():
    anns = [(1, 1, (0, 0, 50, 50), 1024.0, 0), (1, 1, (60, 0, 10, 10), 9216.0, 0)]
    ev = CocoRef(dataset([(1, 100, 100)], anns)).evaluate([])
    r = ev["recall"][0, 0]                     # [area, maxDet]: 0 where ground truth exists, -1 where none
    assert r[0].tolist() == [0, 0, 0] and r[1].tolist() == [0, 0, 0] and r[2].tolist() == [0, 0, 0]
    assert r[3].tolist() == [0, 0, 0]
    ev = CocoRef(dataset([(1, 100, 100)], anns[:1])).evaluate([])
    assert ev["recall"][0, 0, :, 0].tolist() == [0, 0, 0, -1]  # 1024: small and medium, not large
    assert np.all(ev["precision"][:, :, 0, :3] == 0)


def test_equal_iou_goes_to_the_later_box_and_threshold_is_inclusive():
    ious = np.array([[0.5, 0.5]])
    assert match_literal(ious, [0, 0], [0, 0], 0.5) == [1]
    assert match_literal(np.array([[0.5 - 1e-12, 0.4]]), [0, 0], [0, 0], 0.5) == [-1]
    assert match_literal(np.array([[1.0]]), [0], [0], 0.95) == [0]
    # 1 - 1e-10 caps the start, so an IoU of exactly 1 still matches at any threshold
    assert match_literal(np.array([[1.0 - 1e-10]]), [0], [0], 1.0) == [0]


def test_crowd_box_matches_twice_and_is_ignored():
    anns = [(1, 1, (0, 0, 40, 40), 1600.0, 1), (1, 1, (60, 60, 20, 20), 400.0, 0)]
    dets = [det(1, (0, 0, 20, 20), 0.9), det(1, (20, 20, 20, 20), 0.8), det(1, (60, 60, 20, 20), 0.7)]
    ev = CocoRef(dataset([(1, 100, 100)], anns)).evaluate(dets)
    # both crowd hits (IoU 400 / 400 = 1) are ignored: the ranked sequence is [ig, ig, TP], npig = 1
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 1.0 / (1.0 + EPS))
    assert np.all(ev["recall"][:, 0, 0, 2] == 1.0)
    # maxDets 1: only the first detection (a crowd hit) remains
    assert np.all(ev["recall"][:, 0, 0, 0] == 0.0) and np.all(ev["precision"][:, 1:, 0, 0, 0] == 0.0)


def test_regular_match_hides_a_better_crowd_box():
    ious = np.array([[0.6, 0.9]])              # sorted order: regular (non-ignored), then crowd (ignored)
    assert match_literal(ious, [0, 1], [0, 1], 0.5) == [0]
    assert match_literal(ious, [0, 1], [0, 1], 0.7) == [1]
    anns = [(1, 1, (0, 0, 10, 10), 100.0, 1), (1, 1, (0, 0, 10, 12), 120.0, 0)]   # crowd first in the file
    ev = CocoRef(dataset([(1, 100, 100)], anns)).evaluate([det(1, (0, 0, 10, 10), 0.5)])
    assert ev["recall"][0, 0, 0, 2] == 1.0     # IoU 100 / 120 with the regular box: a TP at 0.5 ...
    assert ev["recall"][9, 0, 0, 2] == 0.0     # ... and at 0.95 the crowd box (IoU 1) takes it: ignored, no FP
    assert np.all(ev["precision"][9, :, 0, 0, 2] == 0.0)


def test_unmatched_detection_outside_the_area_range_is_ignored():
    anns = [(1, 1, (0, 0, 10, 10), 100.0, 0)]
    dets = [det(1, (50, 50, 40, 40), 0.9), det(1, (0, 0, 10, 10), 0.8)]     # a large FP, then the small TP
    ev = CocoRef(dataset([(1, 100, 100)], anns)).evaluate(dets)
    small, all_ = ev["precision"][0, :, 0, 1, 2], ev["precision"][0, :, 0, 0, 2]
    assert np.all(small == 1.0 / (1.0 + EPS))  # area 1600 is outside "small": ignored there
    assert np.all(all_ == 1.0 / (2.0 + EPS))   # but an FP in "all": pr = [0, 1/2]


def test_ties_across_images_rank_in_sorted_image_id_order():
    anns = [(7, 1, (0, 0, 10, 10), 100.0, 0)]
    ds = dataset([(7, 100, 100), (3, 100, 100)], anns)         # listed out of order
    ev = CocoRef(ds).evaluate([det(7, (0, 0, 10, 10), 0.5), det(3, (0, 0, 10, 10), 0.5)])
    # image 3's FP ranks first: rc = [0, 1], pr = [0, 1/2]
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 1.0 / (2.0 + EPS))
    ds = dataset([(7, 100, 100), (30, 100, 100)], anns)
    ev = CocoRef(ds).evaluate([det(30, (0, 0, 10, 10), 0.5), det(7, (0, 0, 10, 10), 0.5)])
    assert np.all(ev["precision"][:, :, 0, 0, 2] == 1.0 / (1.0 + EPS))


def test_searchsorted_lookup_and_envelope():
    # npig 4; ranked TP, FP, TP: rc = [.25, .25, .5], pr = [1, 1/2, 2/3] -> envelope [1, 2/3, 2/3]
    anns = [(1, 1, (20 * k, 0, 10, 10), 100.0, 0) for k in range(4)]
    dets = [det(1, (0, 0, 10, 10), 0.9), det(1, (0, 50, 10, 10), 0.8), det(1, (20, 0, 10, 10), 0.7)]
    ev = CocoRef(dataset([(1, 100, 100)], anns)).evaluate(dets)
    p = ev["precision"][0, :, 0, 0, 2]
    rc = np.array([1, 1, 2]) / 4
    pr = np.array([1, 1, 2]) / (np.array([0, 1, 1]) + np.array([1, 1, 2]) + EPS)
    env = np.maximum.accumulate(pr[::-1])[::-1]
    idx = np.searchsorted(rc, coco_ref.REC_THRS, side="left")
    want = np.where(idx < 3, env[np.minimum(idx, 2)], 0.0)
    assert np.array_equal(p, want) and p[0] == env[0] and p[26] == env[2] and p[51] == 0.0
    assert ev["recall"][0, 0, 0, 2] == 0.5 and ev["recall"][0, 0, 0, 0] == 0.25


def test_class_without_ground_truth_is_minus_one_and_nan_per_class():
    ds = dataset([(1, 100, 100)], [(1, 5, (0, 0, 10, 10), 100.0, 0)], cats=(5, 2))
    ev = CocoRef(ds).evaluate([det(1, (0, 0, 10, 10), 0.5, cat=2)])
    assert np.all(ev["precision"][:, :, 0] == -1) and np.all(ev["recall"][:, 0] == -1)      # category 2: index 0
    assert np.isnan(ev["ap_per_class"][0]) and ev["ap_per_class"][1] == 0.0


@pytest.mark.parametrize("seed", range(6))
def test_two_tier_form_equals_the_literal_loop(seed):
    rng = np.random.default_rng(seed)
    for _ in range(400):
        D, G = int(rng.integers(1, 8)), int(rng.integers(1, 8))
        ious = rng.choice([0.0, 0.5, 0.55, 0.75, 0.9, 1.0 - 1e-10, 1.0], (D, G))
        crowd = rng.random(G) < 0.3
        ignored = crowd | (rng.random(G) < 0.3)
        order = np.argsort(ignored, kind="mergesort")
        ig, cr, io = ignored[order].astype(int), crowd[order].astype(int), ious[:, order]
        for t in coco_ref.IOU_THRS:
            assert match_literal(io, ig, cr, t) == match_two_tier(io, ig, cr, t)


def _write(tmp_path, ds, name="inst.json"):
    p = tmp_path / name
    p.write_text(json.dumps(ds))
    return str(p)


def test_loader_sorts_and_packs(tmp_path):
    from k210_yolo_framework_b200.evaluate import load_coco_annotations
    ds = dataset([(9, 20, 30), (2, 40, 50), (5, 60, 70)],
                 [(9, 8, (1, 2, 3, 4), 10.0, 0), (2, 3, (5, 6, 7, 8), 20.0, 1), (9, 3, (9, 10, 11, 12), 30.0, 0)],
                 cats=(8, 3))
    images, cats, gt = load_coco_annotations(_write(tmp_path, ds))
    assert images == [(2, "2.jpg", (40, 50)), (5, "5.jpg", (60, 70)), (9, "9.jpg", (20, 30))]
    assert cats == [3, 8] and gt.category_ids == (3, 8)
    assert gt.offsets.tolist() == [0, 1, 1, 3]
    assert gt.rows.tolist() == [[0, 5, 6, 7, 8, 20, 1], [1, 1, 2, 3, 4, 10, 0], [0, 9, 10, 11, 12, 30, 0]]


@pytest.mark.parametrize("bad,match", [("category", "unknown category"), ("image", "not listed"), ("id0", "is 0"),
                                       ("dup", "repeated"), ("crowd", "iscrowd")])
def test_loader_refuses_malformed_files(tmp_path, bad, match):
    from k210_yolo_framework_b200.evaluate import load_coco_annotations
    ds = dataset([(1, 10, 10)], [(1, 1, (0, 0, 1, 1), 1.0, 0), (1, 1, (0, 0, 2, 2), 4.0, 0)])
    a = ds["annotations"][1]
    if bad == "category":
        a["category_id"] = 4
    elif bad == "image":
        a["image_id"] = 2
    elif bad == "id0":
        a["id"] = 0
    elif bad == "dup":
        a["id"] = 1
    else:
        a["iscrowd"] = 2
    with pytest.raises(ValueError, match=match):
        load_coco_annotations(_write(tmp_path, ds))


def test_results_file_round_trip_gives_the_same_stats(tmp_path):
    from k210_yolo_framework_b200.evaluate import coco_results
    ds, dets, counts = synthetic_coco(11, 12, 5, 20, mean_dets=3)
    ids = sorted(im["id"] for im in ds["images"])
    cats = sorted(c["id"] for c in ds["categories"])
    res = coco_results(dets, counts, ids, cats)
    assert res == records_to_results(dets, counts, ids, cats)
    path = tmp_path / "results.json"
    path.write_text(json.dumps(res))
    loaded = json.loads(path.read_text())
    assert loaded == res                      # every float64 survives the text form
    a, b = CocoRef(ds).evaluate(res), CocoRef(ds).evaluate(loaded)
    assert np.array_equal(a["precision"], b["precision"]) and np.array_equal(a["stats"], b["stats"])
    assert a["stats"][0] > 0


def test_summary_text_and_stats_restate_summarize():
    from k210_yolo_framework_b200.evaluate import coco_stats, coco_summary
    ds, dets, counts = synthetic_coco(12, 10, 4, 20, mean_dets=3)
    ids = sorted(im["id"] for im in ds["images"])
    ev = CocoRef(ds).evaluate(records_to_results(dets, counts, ids, sorted(c["id"] for c in ds["categories"])))
    assert np.array_equal(coco_stats(ev["precision"], ev["recall"]), ev["stats"])
    lines = coco_summary(ev["stats"])
    assert lines == ev["lines"] and len(lines) == 12
    assert lines[0] == f" Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = {ev['stats'][0]:0.3f}"
    assert lines[2].startswith(" Average Precision  (AP) @[ IoU=0.75      | area=   all | maxDets=100 ]")
    assert lines[9].startswith(" Average Recall     (AR) @[ IoU=0.50:0.95 | area= small | maxDets=100 ]")
    assert coco_summary([-1] * 12)[6].endswith("maxDets=  1 ] = -1.000")


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_matches_pycocotools(tmp_path, seed):
    pytest.importorskip("pycocotools")
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval
    ds, dets, counts = synthetic_coco(seed, 25, 6, 120, mean_dets=5, empty_every=6)
    ids = sorted(im["id"] for im in ds["images"])
    res = records_to_results(dets, counts, ids, sorted(c["id"] for c in ds["categories"]))
    gt = COCO(_write(tmp_path, ds))
    ce = COCOeval(gt, gt.loadRes(res), "bbox")
    ce.evaluate()
    ce.accumulate()
    ce.summarize()
    want = CocoRef(ds).evaluate(res)
    assert np.array_equal(ce.eval["precision"], want["precision"])
    assert np.array_equal(ce.eval["recall"], want["recall"])
    assert np.array_equal(ce.stats, want["stats"])
