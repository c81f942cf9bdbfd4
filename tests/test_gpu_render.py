"""GPU rendering (csrc/render.cu) against draw.draw_detections, pixel for pixel, and the rendering path of the pipelines and
serve.py --draw against PIL's draw_detections + save."""
import io
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from PIL import Image

from conftest import GOLDEN
from render_ref import render_ref
from k210_yolo_framework_b200.detect import DET_DTYPE
from k210_yolo_framework_b200.draw import draw_detections
from k210_yolo_framework_b200.helper import _COLORMAP, read_image
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline
from k210_yolo_framework_b200.render import LabelAtlas, render_detections_device

FONT = "missing.otf"      # PIL's default font, as draw_detections falls back to it


def pack(found_per_image, C, K):
    """to_host tuples per image -> device dets int32 [n, C, K, 6], counts int32 [n, C]."""
    n = len(found_per_image)
    rec = np.zeros((n, C, K), DET_DTYPE)
    counts = np.zeros((n, C), np.int32)
    for i, found in enumerate(found_per_image):
        for c, idx, s, t, l, b, r in found:
            k = counts[i, c]
            rec[i, c, k] = (t, l, b, r, s, idx)
            counts[i, c] += 1
    dets = torch.from_numpy(rec.view(np.int32).reshape(n, C, K, 6).copy()).cuda()
    return dets, torch.from_numpy(counts).cuda()


def f32(found):
    """Records as the device holds them: every coordinate and score a float32 value (draw_detections formats what it is given)."""
    return [(c, i) + tuple(float(np.float32(v)) for v in rest) for c, i, *rest in found]


def render_gpu(imgs, found_per_image, C=20, K=40, atlas=None):
    atlas = atlas or LabelAtlas(C, FONT)
    views = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in imgs]
    dets, counts = pack(found_per_image, C, K)
    render_detections_device(views, dets, counts, atlas)
    torch.cuda.synchronize()
    return [v.cpu().numpy() for v in views]


def assert_pil(imgs, found_per_image, C=20, K=40):
    found_per_image = [f32(f) for f in found_per_image]
    got = render_gpu(imgs, found_per_image, C, K)
    for i, (g, x, f) in enumerate(zip(got, imgs, found_per_image)):
        ref = np.array(draw_detections(x, f, _COLORMAP, font_path=FONT))
        assert np.array_equal(g, ref), (i, x.shape, int((g != ref).any(-1).sum()))


def seeded(h, w, n, C, seed):
    from test_render_host import seeded_records
    return seeded_records(h, w, n, C, seed)


def test_dog_golden_records(dog_u8, dog_golden):
    found = [tuple(d) for d in dog_golden["keras"]["detections"]]
    assert_pil([dog_u8], [found])


def test_seeded_records_mixed_sizes_thickness_edges():
    shapes = [(224, 320), (375, 500), (1080, 1920), (17, 40), (600, 333)]
    imgs = [np.random.default_rng(i).integers(0, 256, s + (3,), dtype=np.uint8) for i, s in enumerate(shapes)]
    found = [seeded(h, w, 30, 20, 7 * i) for i, (h, w) in enumerate(shapes)]
    assert (1080 + 1920) // 300 == 10
    assert_pil(imgs, found)


def test_overlapping_classes_scores_and_label_edges():
    img = np.full((300, 400, 3), 90, np.uint8)
    found = [(0, 0, 0.005, 50.0, 50.0, 200.0, 300.0), (0, 1, 0.125, 60.4, 60.5, 210.0, 310.0), (3, 2, 0.995, 55.0, 40.0, 150.0, 250.0),
             (7, 3, 1.0, 290.0, 380.0, 299.0, 399.0),      # label runs off the right and bottom edges
             (19, 4, float(np.float32(0.7)), -20.0, -30.0, 500.0, 600.0)]
    assert_pil([img], [found])


def test_every_class_no_records_and_top_at_bottom():
    img = np.full((150, 500, 3), 180, np.uint8)
    found = [(c, 0, float(np.float32(((c * 37) % 101) / 100)), 10.0, 5.0 + 6 * c, 120.0, 30.0 + 6 * c) for c in range(80)]
    bottom = f32([(5, 0, 0.5, 150.0, 20.0, 160.0, 60.0), (6, 1, 0.6, 149.6, 100.0, 149.7, 190.0)])   # top >= h: label above the top
    low = np.full((150, 200, 3), 60, np.uint8)          # one ring: the clipped boxes have no second ring to cross
    got = render_gpu([img, img, low], [found, [], bottom], C=80, K=4)
    assert np.array_equal(got[0], np.array(draw_detections(img, found, _COLORMAP, font_path=FONT)))
    assert np.array_equal(got[1], img)
    assert np.array_equal(got[2], np.array(draw_detections(low, bottom, _COLORMAP, font_path=FONT)))


def test_crossing_rings_stop_at_the_first_crossing_ring():
    img = np.full((1200, 1500, 3), 30, np.uint8)      # 9 rings
    found = f32([(1, 0, 0.9, 100.0, 100.0, 400.0, 101.0), (2, 1, 0.8, 500.0, 200.0, 503.0, 700.0), (4, 2, 0.4, 800.0, 900.0, 800.0, 900.0)])
    with pytest.raises(ValueError):
        draw_detections(img, found[:1], _COLORMAP, font_path=FONT)
    atlas = LabelAtlas(20, FONT)
    got = render_gpu([img], [found], atlas=atlas)[0]
    assert np.array_equal(got, render_ref(img, found, _COLORMAP, atlas.host(1200)))


# -- the pipelines ------------------------------------------------------------------------------------------------------
IN_HW = (224, 320)


def make_pipe(voc_anchors, golden_weights, laned=False):
    args = ("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 4, 0.3, 0.3)
    pipe = LanedPipeline(2, *args) if laned else DetectionPipeline(*args)
    if laned:
        pipe.set_weights(golden_weights)
    else:
        pipe.engine.set_weights(golden_weights)
    return pipe


def jpeg(img, q=90):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=q)
    return b.getvalue()


def png(img):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "PNG")
    return b.getvalue()


def batches(dog_u8, people_u8):
    rng = np.random.default_rng(3)
    noise = rng.integers(0, 256, (200, 260, 3), dtype=np.uint8)
    return [[jpeg(dog_u8), png(people_u8), noise, jpeg(people_u8, 75)],
            [people_u8, jpeg(noise), png(dog_u8)],
            [jpeg(dog_u8[:, ::-1].copy()), dog_u8],
            [png(noise), jpeg(people_u8), jpeg(dog_u8, 50), people_u8]]


def as_pixels(item):
    return item if isinstance(item, np.ndarray) else read_image(io.BytesIO(bytes(item)))


@pytest.mark.parametrize("laned", [False, True])
def test_pipeline_rendering(voc_anchors, golden_weights, dog_u8, people_u8, laned):
    bs = batches(dog_u8, people_u8)

    def run(render):
        pipe = make_pipe(voc_anchors, golden_weights, laned)
        if render:
            pipe.enable_rendering(quality=85, font_path=FONT)
        out, pending = [], []
        for b in bs:                                        # two batches in flight
            pending.append(pipe.submit_images(b))
            if len(pending) == 2:
                t = pending.pop(0)
                recs = DetectionPipeline.records(*pipe.collect(t))
                out.append((recs, pipe.rendered(t) if render else None))
        for t in pending:
            recs = DetectionPipeline.records(*pipe.collect(t))
            out.append((recs, pipe.rendered(t) if render else None))
        return out

    plain, drawn = run(False), run(True)
    assert [r for r, _ in plain] == [r for r, _ in drawn]
    for b, (recs, files) in zip(bs, drawn):
        assert len(files) == len(b)
        for item, rec, f in zip(b, recs, files):
            ref = io.BytesIO()
            draw_detections(as_pixels(item), rec, _COLORMAP, font_path=FONT).save(ref, "JPEG", quality=85)
            assert f == ref.getvalue()
    assert any(len(r) for recs, _ in drawn for r in recs)


def test_enable_rendering_refuses_more_classes_than_colours(voc_anchors):
    pipe = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 2)
    with pytest.raises(ValueError):
        pipe.enable_rendering(colormap=_COLORMAP[:10])
    with pytest.raises(RuntimeError):
        pipe.rendered(0)


def test_serve_draw(tmp_path, golden_weights, dog_u8, people_u8):
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    for i, b in enumerate(batches(dog_u8, people_u8)):
        for j, item in enumerate(b):
            if isinstance(item, np.ndarray):
                Image.fromarray(item).save(d / f"im{i}{j}.bmp")
            else:
                (d / f"im{i}{j}{'.jpg' if item[:2] == b'\xff\xd8' else '.png'}").write_bytes(item)
    common = [str(ckpt), str(d), "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", "4", "--obj_thresh", "0.3",
              "--iou_thresh", "0.3", "--decode_threads", "2"]
    lines = {}
    for draw in (False, True):
        out = str(tmp_path / f"out{int(draw)}.jsonl")
        args = serve.build_parser().parse_args(common + ["--out", out] + (["--draw", str(tmp_path / "drawn"), "--draw_quality", "80"] if draw else []))
        with open(out, "w") as fh:
            assert serve.serve(args, fh) == 13
        lines[draw] = open(out).read()
    assert lines[False] == lines[True]
    assert sorted(os.listdir(tmp_path / "drawn")) == sorted(os.path.splitext(f)[0] + ".jpg" for f in os.listdir(d))
    for line in lines[True].splitlines():
        rec = json.loads(line)
        found = [(x["class"], x["index"], x["score"], *x["box_tlbr"]) for x in rec["detections"]]
        ref = io.BytesIO()
        draw_detections(read_image(rec["image"]), found, _COLORMAP).save(ref, "JPEG", quality=80)
        stem = os.path.splitext(os.path.basename(rec["image"]))[0]
        assert (tmp_path / "drawn" / (stem + ".jpg")).read_bytes() == ref.getvalue(), stem
