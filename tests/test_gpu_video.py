"""Video on the GPU: DHT-less baseline frames decode to PIL's pixels; serve.py over a Motion-JPEG AVI and an mp4v video gives the
records and JSON lines of submitting each frame as an image; the --draw AVI holds the drawn frames PIL would write; 2 GPUs give
what 1 gives."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from test_video import _img, _pil, build_avi, strip_dht

pytestmark = pytest.mark.gpu


def _cv2(img, factor, rst=0):
    import cv2
    ok, buf = cv2.imencode(".jpg", img[..., ::-1].copy(), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, factor),
                                                          cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
    assert ok
    return buf.tobytes()


def _gray(img, **kw):
    from PIL import Image
    return _pil(np.asarray(Image.fromarray(img).convert("L")), **kw)


def _layout_files():
    out = []
    for k, (h, w) in enumerate([(48, 64), (37, 53), (120, 97)]):
        img = _img(h, w, seed=k)
        for rst in (0, 2):
            kw = {"restart_marker_blocks": rst} if rst else {}
            out += [_pil(img, quality=80, subsampling=0, **kw), _pil(img, quality=90, subsampling=1, **kw),
                    _pil(img, quality=70, subsampling=2, **kw), _gray(img, quality=85, **kw),
                    _cv2(img, "IMWRITE_JPEG_SAMPLING_FACTOR_440", rst), _cv2(img, "IMWRITE_JPEG_SAMPLING_FACTOR_411", rst)]
    return out


def test_dht_less_frames_decode_to_pil_pixels():
    from k210_yolo_framework_b200 import preprocess
    from k210_yolo_framework_b200.helper import read_image
    files = [strip_dht(f) for f in _layout_files()]
    assert all(preprocess.gpu_decodable(f) for f in files)
    got = preprocess.decode_jpeg_batch(files)
    for i, (f, g) in enumerate(zip(files, got)):
        np.testing.assert_array_equal(g.cpu().numpy(), read_image(io.BytesIO(f)), err_msg=f"file {i}")


def test_padded_and_two_field_payloads_give_pil_pixels_of_the_uncut_payload(tmp_path):
    from k210_yolo_framework_b200 import preprocess, video
    from k210_yolo_framework_b200.helper import read_image
    a, b = strip_dht(_pil(_img(seed=1), quality=80, subsampling=1)), strip_dht(_pil(_img(seed=2), quality=60))
    stored = [a + bytes(9), a + b, b + b"\xff" * 3, a + b"\x00\x00\xff\xd8"]
    p = tmp_path / "v.avi"
    p.write_bytes(build_avi(stored))
    v = video.open_video(str(p))
    frames = [v.frame_bytes(k) for k in range(v.n_frames)]
    assert all(preprocess.gpu_decodable(f) for f in frames)
    assert not any(preprocess.gpu_decodable(stored[k]) for k in (0, 2, 3))     # uncut, these would go to PIL
    for f, s, g in zip(frames, stored, preprocess.decode_jpeg_batch(frames)):
        np.testing.assert_array_equal(g.cpu().numpy(), read_image(io.BytesIO(s)))


# ---------------------------------------------------------------------------------------------------------------------
# serve.py
# ---------------------------------------------------------------------------------------------------------------------
def _scene(k, h=240, w=320):
    """Frame k of a moving scene: the golden dog photo panned across a background."""
    dog = np.load(os.path.join(GOLDEN, "dog_u8.npy"))
    out = _img(h, w, seed=100 + k)
    dh, dw = min(dog.shape[0], h), min(dog.shape[1], w - 40)
    x0 = (7 * k) % 40
    out[:dh, x0:x0 + dw] = dog[:dh, :dw]
    return out


def _args(tmp_path, images, batch=4, **kw):
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    from k210_yolo_framework_b200.yolonet import load_npz_weights
    ckpt = tmp_path / "model.h5"
    if not ckpt.exists():
        save_keras_weights(str(ckpt), load_npz_weights(os.path.join(GOLDEN, "yolo_mobilev1_075_voc_weights.npz")))
    argv = [str(ckpt), str(images), "--anchors", os.path.join(GOLDEN, "voc_anchor.npy"), "--batch", str(batch),
            "--obj_thresh", "0.3"]
    for k, v in kw.items():
        argv += [f"--{k}"] + ([] if v is True else [str(x) for x in (v if isinstance(v, (list, tuple)) else [v])])
    return serve.build_parser().parse_args(argv)


def _serve(args):
    import serve
    out = io.StringIO()
    n = serve.serve(args, out)
    return n, out.getvalue().splitlines()


def _image_lines(tmp_path, images, args_kw, batch=4):
    """serve.py's lines for each frame submitted as an image file (PNG files of the given pixels, or the JPEG bytes)."""
    d = tmp_path / "frames"
    d.mkdir(exist_ok=True)
    for f in d.iterdir():
        f.unlink()
    for k, im in enumerate(images):
        if isinstance(im, bytes):
            (d / f"{k:04d}.jpg").write_bytes(im)
        else:
            from PIL import Image
            Image.fromarray(im).save(d / f"{k:04d}.png")
    n, lines = _serve(_args(tmp_path, d, batch, **args_kw))
    return [json.loads(l)["detections"] for l in lines]


def _mjpeg_video(tmp_path, n=11):
    frames = [strip_dht(_pil(_scene(k), quality=90, subsampling=1)) for k in range(n)]
    stored = [f + bytes(k % 3) for k, f in enumerate(frames)]        # some padded, as cameras write them
    stored[4] = frames[4] + frames[5]                                 # a two-field frame
    stored.insert(6, b"")                                             # a dropped frame
    p = tmp_path / "cam.avi"
    p.write_bytes(build_avi(stored, w=320, h=240, scale=1001, rate=30000))
    return p, stored


@pytest.mark.parametrize("kw", [{}, {"tiles": (1, 2), "flip": True}])
def test_serve_mjpeg_avi_equals_frames_as_images(tmp_path, kw):
    from k210_yolo_framework_b200 import video
    from k210_yolo_framework_b200.helper import read_image
    p, stored = _mjpeg_video(tmp_path)
    batch = 4 if not kw else 12
    n, lines = _serve(_args(tmp_path, p, batch, **kw))
    recs = [json.loads(l) for l in lines]
    payloads = [s for s in stored if s]
    assert n == len(payloads) == 11          # 11 frames: a short final batch
    positions = [i for i, s in enumerate(stored) if s]
    assert [r["frame"] for r in recs] == positions and all(r["video"] == str(p) for r in recs)
    assert [r["time"] for r in recs] == [i * 1001 / 30000 for i in positions]
    ref = _image_lines(tmp_path, [read_image(io.BytesIO(s)) for s in payloads], kw, batch)     # PIL's pixels of each chunk
    assert [r["detections"] for r in recs] == ref
    assert sum(len(r) for r in ref) > 0
    v = video.open_video(str(p))
    assert all(video.cut_frame(s) == v.frame_bytes(k) for k, s in enumerate(payloads))


def test_serve_mp4v_equals_frames_as_images(tmp_path):
    import cv2
    p = str(tmp_path / "clip.mp4")
    w = cv2.VideoWriter(p, cv2.CAP_FFMPEG, cv2.VideoWriter_fourcc(*"mp4v"), 24.0, (320, 240))
    assert w.isOpened()
    for k in range(9):
        w.write(_scene(k)[..., ::-1].copy())
    w.release()
    cap = cv2.VideoCapture(p, cv2.CAP_FFMPEG)
    pixels = []
    while True:
        ok, bgr = cap.read()
        if not ok:
            break
        pixels.append(np.ascontiguousarray(bgr[..., ::-1]))
    assert len(pixels) == 9
    for kw in ({}, {"tiles": (1, 2), "flip": True}):
        batch = 4 if not kw else 12
        n, lines = _serve(_args(tmp_path, p, batch, decode_threads=3, **kw))
        recs = [json.loads(l) for l in lines]
        assert n == 9 and [r["frame"] for r in recs] == list(range(9)) and [r["time"] for r in recs] == [k / 24 for k in range(9)]
        assert [r["detections"] for r in recs] == _image_lines(tmp_path, pixels, kw, batch)


def test_serve_draw_writes_the_drawn_frames(tmp_path):
    from k210_yolo_framework_b200 import video
    from k210_yolo_framework_b200.draw import draw_detections
    from k210_yolo_framework_b200.helper import _COLORMAP, read_image
    p, stored = _mjpeg_video(tmp_path, 7)
    out = tmp_path / "drawn"
    n, lines = _serve(_args(tmp_path, p, 4, draw=str(out), draw_quality=85))
    v = video.open_video(str(out / "cam.avi"))
    src = video.open_video(str(p))
    assert v.n_frames == n == 7 and v.fps == pytest.approx(30000 / 1001) and v.frame_hw == (240, 320)
    assert sum(len(json.loads(l)["detections"]) for l in lines) > 0
    for k, line in enumerate(lines):
        found = [(d["class"], d["index"], d["score"], *d["box_tlbr"]) for d in json.loads(line)["detections"]]
        ref = io.BytesIO()
        draw_detections(read_image(io.BytesIO(src.frame_bytes(k))), found, _COLORMAP).save(ref, "JPEG", quality=85)
        assert v.frame_bytes(k) == ref.getvalue(), f"frame {k}"


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


def test_two_gpus_write_what_one_writes(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    p, _ = _mjpeg_video(tmp_path, 13)
    one_dir, two_dir = tmp_path / "one", tmp_path / "two"
    a = _args(tmp_path, p, 4, draw=str(one_dir))
    n, one = _serve(a)
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    argv = [a.ckpt, str(p), "--anchors", a.anchors, "--batch", "4", "--obj_thresh", "0.3", "--draw", str(two_dir)]
    env = dict(os.environ, K2Y_ROOT=ROOT, PYTHONPATH=ROOT, K2Y_OUT=str(tmp_path / "two.jsonl"))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29543", str(script)] + argv, capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert open(tmp_path / "two.jsonl").read().splitlines() == one
    assert (two_dir / "cam.avi").read_bytes() == (one_dir / "cam.avi").read_bytes()
