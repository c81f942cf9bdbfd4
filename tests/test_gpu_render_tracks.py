"""GPU track drawing (k2y_render_tracks) against draw.draw_tracks pixel for pixel, and the track-drawing path of
DetectionPipeline and serve.py --draw_tracks against draw_tracks + PIL's save."""
import io
import json

import numpy as np
import pytest
import torch
from PIL import ImageFont

pytestmark = pytest.mark.gpu

from render_tracks_ref import render_tracks_ref
from test_render_tracks_host import INT32_MAX, seeded_tracks
from k210_yolo_framework_b200.draw import draw_tracks
from k210_yolo_framework_b200.helper import _COLORMAP, read_image
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline
from k210_yolo_framework_b200.render import TrackLabelAtlas, render_tracks_device

FONT = "missing.otf"      # PIL's default font, as draw_tracks falls back to it


def pack(tracks_per_image, C, K):
    """(class, id, top, left, bottom, right) per image -> device counts [n, C], ids [n, C, K], boxes [n, C, K, 4], with
    unused rows poisoned (the kernel must read only k < counts)."""
    n = len(tracks_per_image)
    counts = np.zeros((n, C), np.int32)
    ids = np.full((n, C, K), 7, np.int32)
    boxes = np.full((n, C, K, 4), 5.0, np.float32)
    for i, tracks in enumerate(tracks_per_image):
        for c, tid, *box in tracks:
            k = counts[i, c]
            ids[i, c, k], boxes[i, c, k] = tid, box
            counts[i, c] += 1
    return tuple(torch.from_numpy(a).cuda() for a in (counts, ids, boxes))


def render_gpu(imgs, tracks_per_image, C=80, K=40, atlas=None, colormap=None):
    atlas = atlas or TrackLabelAtlas(FONT)
    views = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in imgs]
    render_tracks_device(views, *pack(tracks_per_image, C, K), atlas, colormap)
    torch.cuda.synchronize()
    return [v.cpu().numpy() for v in views]


def test_seeded_tracks_mixed_sizes_and_ids():
    shapes = [(224, 320), (375, 500), (1080, 1920), (17, 40), (600, 333), (720, 1280)]
    imgs = [np.random.default_rng(i).integers(0, 256, s + (3,), dtype=np.uint8) for i, s in enumerate(shapes)]
    tracks = [seeded_tracks(h, w, 36, 80, 11 * i) for i, (h, w) in enumerate(shapes)]
    assert {-1, 1, INT32_MAX} <= {t[1] for ts in tracks for t in ts}
    got = render_gpu(imgs, tracks)
    for i, (g, x, t) in enumerate(zip(got, imgs, tracks)):
        ref = np.array(draw_tracks(x, t, _COLORMAP, font_path=FONT))
        assert np.array_equal(g, ref), (i, x.shape, int((g != ref).any(-1).sum()))


def test_no_tracks_all_lost_and_a_short_colormap():
    img = np.full((200, 300, 3), 120, np.uint8)
    lost = [(c, -1, 10.0, 10.0, 100.0, 100.0) for c in range(3)]
    some = [(0, 3, 20.0, 20.0, 120.0, 150.0), (2, 4, 30.0, 40.0, 130.0, 200.0), (2, 1000000000, 50.0, 60.0, 150.0, 290.0)]
    cmap = _COLORMAP[:3]
    got = render_gpu([img, img, img], [[], lost, some], C=3, K=6, colormap=cmap)
    assert np.array_equal(got[0], img) and np.array_equal(got[1], img)
    assert np.array_equal(got[2], np.array(draw_tracks(img, some, cmap, font_path=FONT)))


def test_crossing_rings_stop_at_the_first_crossing_ring():
    img = np.full((1200, 1500, 3), 30, np.uint8)      # 9 rings
    tracks = [(1, 5, 100.0, 100.0, 400.0, 101.0), (2, 77, 500.0, 200.0, 503.0, 700.0), (4, INT32_MAX, 800.0, 900.0, 800.0, 900.0)]
    with pytest.raises(ValueError):
        draw_tracks(img, tracks[:1], _COLORMAP, font_path=FONT)
    atlas = TrackLabelAtlas(FONT)
    got = render_gpu([img], [tracks], C=20, atlas=atlas)[0]
    assert np.array_equal(got, render_tracks_ref(img, tracks, _COLORMAP, atlas.host(1200)))


def test_truetype_sizes_in_one_launch_blend_overlapping_glyphs(tmp_path):
    """The default font's TrueType bytes at 7, 11, 21 and 32 px (image heights 224, 375, 700, 1080), one atlas per image in
    one launch, with labels whose glyph masks overlap: at 7 and 11 px "#4444"-style labels differ between the blend and
    max, and the kernel must draw the blend, as draw_tracks does."""
    ttf = tmp_path / "default.ttf"
    ttf.write_bytes(ImageFont.load_default().font_bytes)
    atlas = TrackLabelAtlas(str(ttf))
    shapes = [(224, 320), (375, 500), (700, 1000), (1080, 1920)]
    ids = [4444, 44444, INT32_MAX, 404, 4747, 1111111111, -1, 7]
    imgs, tracks = [], []
    for i, (h, w) in enumerate(shapes):
        imgs.append(np.random.default_rng(40 + i).integers(0, 256, (h, w, 3), dtype=np.uint8))
        u = h / 224           # a grid of boxes, each label clear of the others
        grid = [(c, ids[c % len(ids)], float(np.float32(10 + 60 * u * (c // 3))), float(np.float32(5 + 105 * u * (c % 3))),
                 float(np.float32(10 + 60 * u * (c // 3) + 50 * u)), float(np.float32(5 + 105 * u * (c % 3) + 95 * u)))
                for c in range(9)]
        tracks.append(grid + [t for t in seeded_tracks(h, w, 12, 80, 70 + i) if t[0] >= 9])
    assert len({atlas.device(h, torch.device("cuda")).data_ptr() for h, _ in shapes}) == 4
    got = render_gpu(imgs, tracks, atlas=atlas)
    blend_differs = []
    for i, (g, x, t) in enumerate(zip(got, imgs, tracks)):
        ref = np.array(draw_tracks(x, t, _COLORMAP, font_path=str(ttf)))
        assert np.array_equal(g, ref), (i, x.shape, int((g != ref).any(-1).sum()))
        by_max = render_tracks_ref(x, t, _COLORMAP, atlas.host(x.shape[0]), blend="max")
        blend_differs.append(int((by_max != ref).any(-1).sum()))
    assert blend_differs[0] > 0 and blend_differs[1] > 0, blend_differs


def test_render_tracks_device_refuses_bad_layouts():
    img = [torch.zeros((20, 20, 3), dtype=torch.uint8, device="cuda")]
    counts, ids, boxes = pack([[]], 4, 3)
    atlas = TrackLabelAtlas(FONT)
    for bad in [(counts, ids.float(), boxes), (counts, ids, boxes[..., :3].contiguous()), (counts, ids[:, :3], boxes),
                (counts.cpu(), ids, boxes), (counts[:, :2], ids, boxes)]:
        with pytest.raises(ValueError):
            render_tracks_device(img, *bad, atlas)
    with pytest.raises(ValueError):
        render_tracks_device(img, *pack([[]], 81, 1), atlas)


# -- the pipeline and serve.py ------------------------------------------------------------------------------------------
def frame_tracks(ids, boxes, counts):
    """One frame's (class, id, top, left, bottom, right) in tracks() order."""
    C, K = ids.shape
    return [(c, int(ids[c, k]), *(float(v) for v in boxes[c, k])) for c in range(C) for k in range(min(int(counts[c]), K))]


def scene_batches():
    from test_gpu_video import _scene
    from test_video import _pil
    rng = np.random.default_rng(5)
    # (images, frames, streams): two streams interleaved, one image past the frames, frames of two sizes, a JPEG file
    out, pos = [], [0, 0]
    for b in range(6):
        imgs, frames, streams = [], [], []
        for j in range(4):
            s = (b + j) % 2
            if b == 3 and j == 3:
                imgs.append(rng.integers(0, 256, (200, 260, 3), dtype=np.uint8))      # not a frame: encoded undrawn
                continue
            img = _scene(pos[s] + 9 * s) if s == 0 else _scene(pos[s] + 9 * s, 300, 400)
            imgs.append(_pil(img, quality=92) if j == 1 else img)
            frames.append(pos[s])
            streams.append(s)
            pos[s] += 1
        out.append((imgs, frames, streams))
    return out


def open_pipe(tmp_path, **track_kw):
    import serve
    from test_gpu_video import _args
    pipe, _, _ = serve.open_pipeline(_args(tmp_path, tmp_path, 4))
    pipe.enable_tracking(streams=2, **track_kw)
    return pipe


@pytest.mark.parametrize("method", ["sort", "ocsort"])
def test_pipeline_draws_the_tracks(tmp_path, method):
    bs = scene_batches()

    def run(draw):
        pipe = open_pipe(tmp_path, method=method)
        if draw:
            pipe.enable_rendering(quality=85, font_path=FONT, tracks=True)
        out, pending = [], []

        def finish(t):
            dets, counts = pipe.collect(t)
            ids, boxes = pipe.tracks(t)
            out.append((DetectionPipeline.records(dets, counts), counts.clone(), ids.clone(), boxes.clone(),
                        pipe.rendered(t) if draw else None))
        for imgs, frames, streams in bs:                    # two batches in flight
            pending.append(pipe.submit_images(imgs, frames=frames, streams=streams))
            if len(pending) == 2:
                finish(pending.pop(0))
        for t in pending:
            finish(t)
        return out

    plain, drawn = run(False), run(True)
    for (r0, c0, i0, b0, _), (r1, c1, i1, b1, _) in zip(plain, drawn):
        assert r0 == r1 and torch.equal(c0, c1) and torch.equal(i0, i1) and torch.equal(b0, b1)
    n_tracks = 0
    for (imgs, frames, _), (_, counts, ids, boxes, files) in zip(bs, drawn):
        assert len(files) == len(imgs)
        for j, (item, f) in enumerate(zip(imgs, files)):
            pixels = item if isinstance(item, np.ndarray) else read_image(io.BytesIO(item))
            tracks = frame_tracks(ids[j].numpy(), boxes[j].numpy(), counts[j].numpy()) if j < len(frames) else []
            n_tracks += sum(t[1] >= 0 for t in tracks)
            ref = io.BytesIO()
            draw_tracks(pixels, tracks, _COLORMAP, font_path=FONT).save(ref, "JPEG", quality=85)
            assert f == ref.getvalue(), (frames, j)
    assert n_tracks > 10


def test_pipeline_refusals(tmp_path, voc_anchors, monkeypatch):
    from k210_yolo_framework_b200 import render
    img = np.full((240, 320, 3), 90, np.uint8)
    pipe = DetectionPipeline("yolo_mobilev1", (224, 320), voc_anchors, 20, 0.75, 2)
    pipe.enable_rendering(tracks=True)
    with pytest.raises(ValueError, match="enable_tracking"):
        pipe.submit_images([img])
    # a font the track atlas refuses is refused by submit_images itself, before anything is enqueued
    pipe = open_pipe(tmp_path)
    pipe.enable_rendering(tracks=True)

    def refuse(font):
        raise ValueError("kerning")
    monkeypatch.setattr(render, "check_track_font", refuse)
    with pytest.raises(ValueError, match="kerning"):
        pipe.submit_images([img], frames=[0], streams=[0])
    assert pipe._submitted == 0 and pipe._track["tracker"].last_positions == [None, None]
    monkeypatch.undo()
    t = pipe.submit_images([img], frames=[0], streams=[0])
    pipe.collect(t)
    assert len(pipe.rendered(t)) == 1
    laned = LanedPipeline(2, "yolo_mobilev1", (224, 320), voc_anchors, 20, 0.75, 2)
    with pytest.raises(NotImplementedError):
        laned.enable_rendering(tracks=True)


def test_serve_two_videos_draw_their_tracks(tmp_path):
    from k210_yolo_framework_b200 import video
    from test_gpu_track_streams import _many_args, _serve_lines, _videos
    vids = _videos(tmp_path, [9, 6])
    out = tmp_path / "drawn"
    lines = [json.loads(l) for l in _serve_lines(_many_args(tmp_path, vids, track=True, draw=str(out), draw_tracks=True,
                                                             draw_quality=80))]
    plain = [json.loads(l) for l in _serve_lines(_many_args(tmp_path, vids, track=True))]
    assert lines == plain
    n_tracks = 0
    for v in vids:
        drawn, src = video.open_video(str(out / f"{v.stem}.avi")), video.open_video(str(v))
        mine = [l for l in lines if l["video"] == str(v)]
        assert drawn.n_frames == src.n_frames == len(mine)
        for k, line in enumerate(mine):
            tracks = [(d["class"], d["track"], *d["track_box_tlbr"]) for d in line["detections"] if d["track"] is not None]
            n_tracks += len(tracks)
            ref = io.BytesIO()
            draw_tracks(read_image(io.BytesIO(src.frame_bytes(k))), tracks, _COLORMAP).save(ref, "JPEG", quality=80)
            assert drawn.frame_bytes(k) == ref.getvalue(), (v, k)
    assert n_tracks > 5
