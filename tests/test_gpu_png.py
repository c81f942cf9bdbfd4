"""GPU PNG decode (csrc/png.cu) against ``read_image`` (PIL): every colour type and depth, encoders and zlib strategies, IDAT
splits, DEFLATE streams zlib never writes (oracle/deflate_ref.py), damaged streams (PIL's outcome decides), and the opt-in
routes through letterbox_batch_device, submit_images and serve.py."""
import io
import json
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import deflate_ref as D
from conftest import GOLDEN
from jpeg_cases import photo
from png_cases import GPU_KINDS, bpp_of, filter_rows, make_png, pil_png, pil_read, png_file, random_rows
from k210_yolo_framework_b200 import preprocess
from k210_yolo_framework_b200.pipeline import DetectionPipeline, LanedPipeline

IN_HW = (224, 320)


def check_batch(files):
    """Decodes `files` in one batch: every file PIL decodes gives PIL's pixels and a zero error word, every file PIL refuses a
    non-zero one.  Returns the status words."""
    got, status = preprocess.decode_png_batch(files, with_status=True)
    for i, f in enumerate(files):
        exp = pil_read(f)
        if isinstance(exp, Exception):
            assert status[i, 0] != 0, (i, exp)
        else:
            assert status[i, 0] == 0, (i, status[i])
            np.testing.assert_array_equal(got[i].cpu().numpy(), exp, err_msg=f"file {i}")
    return status


@pytest.mark.parametrize("kind", GPU_KINDS, ids=[f"ct{c}_d{d}" for c, d in GPU_KINDS])
def test_every_kind_and_size(kind):
    color, depth = kind
    rng = np.random.default_rng(color * 100 + depth)
    sizes = [(1, 1), (1, 37), (37, 1), (13, 29), (7, 333), (64, 3)]
    contents = ["noise", "flat", "photo", "detail"]
    files = [make_png(rng, w, h, color, depth, contents[k % 4]) for k, (h, w) in enumerate(sizes)]
    check_batch(files)


@pytest.mark.parametrize("kind", [(2, 8), (3, 4), (6, 16), (0, 1)])
def test_full_hd(kind):
    rng = np.random.default_rng(7)
    check_batch([make_png(rng, 1920, 1080, *kind, content="photo"), make_png(rng, 1920, 1080, *kind, content="noise", level=1)])


def test_pil_levels_and_cv2():
    imgs = [photo(480, 640, 1), photo(375, 500, 2), photo(100, 131, 3)]
    files = [pil_png(im, compress_level=lv) for im in imgs for lv in (0, 1, 6, 9)]
    cv2 = pytest.importorskip("cv2")
    files += [cv2.imencode(".png", im[..., ::-1])[1].tobytes() for im in imgs]
    check_batch(files)


@pytest.mark.parametrize("strategy", [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED])
def test_zlib_strategies_over_all_filters(strategy):
    rng = np.random.default_rng(strategy)
    files = []
    for color, depth in [(2, 8), (0, 8), (3, 8), (6, 16), (0, 4)]:
        for content in ("photo", "noise"):
            files.append(make_png(rng, 97, 61, color, depth, content, types=(0, 1, 2, 3, 4, 4, 3, 1), strategy=strategy))
            files.append(make_png(rng, 40, 30, color, depth, content, types=tuple(rng.integers(0, 5, 30)), strategy=strategy))
    check_batch(files)


def test_idat_splits():
    rng = np.random.default_rng(3)
    rows = random_rows(rng, 50, 40, 2, 8, "photo")
    stream = zlib.compress(filter_rows(rows, 3, (1, 2, 3, 4, 0)))
    files = [png_file(50, 40, 2, 8, stream, split=list(range(1, len(stream)))),          # 1-byte IDATs
             png_file(50, 40, 2, 8, stream, split=[0, 0, 1, 1, 2, 5, 5, len(stream), len(stream)]),   # empty IDATs
             png_file(50, 40, 2, 8, stream)]
    check_batch(files)


def _grey(w, h, rows_u8):
    """(file builder, raw filtered bytes) of a greyscale 8-bit image whose rows use filter 0."""
    raw = b"".join(b"\x00" + bytes(r) for r in rows_u8)
    return (lambda stream: png_file(w, h, 0, 8, stream)), raw


def _tokenize(raw, dist, max_len=258, via284=False):
    """Literals, plus matches at exactly `dist` wherever at least 3 bytes repeat."""
    out, i = [], 0
    while i < len(raw):
        if i >= dist:
            n = 0
            while n < max_len and i + n < len(raw) and raw[i + n] == raw[i + n - dist]:
                n += 1
            if n >= 3:
                out.append((n, dist, D.VIA_284) if via284 and n == 258 else (n, dist))
                i += n
                continue
        out.append(raw[i])
        i += 1
    return out


def _stream(blocks, raw):
    w = D.BitWriter()
    for k, (kind, tokens, kw) in enumerate(blocks):
        final = k == len(blocks) - 1
        if kind == "stored":
            D.stored(w, bytes(tokens), final)
        elif kind == "fixed":
            D.fixed(w, tokens, final)
        else:
            D.dynamic(w, tokens, final, **kw)
    return D.zlib_wrap(w.getvalue(), raw)


def test_deflate_ref_streams():
    rng = np.random.default_rng(11)
    files = []
    # stored blocks of 0 and 65535 bytes
    build, raw = _grey(255, 300, rng.integers(0, 256, (300, 255), dtype=np.uint8))
    files.append(build(_stream([("stored", b"", {}), ("stored", raw[:65535], {}), ("stored", raw[65535:], {})], raw)))
    # many tiny blocks, fixed and dynamic in turn, and one dynamic block spanning the whole image
    build, raw = _grey(31, 40, rng.integers(0, 4, (40, 31), dtype=np.uint8))
    toks = _tokenize(raw, 31 + 1)
    tiny = [("fixed" if k % 2 else "dynamic", toks[k:k + 3], {}) for k in range(0, len(toks), 3)]
    files += [build(_stream(tiny, raw)), build(_stream([("dynamic", toks, {})], raw)), build(_stream([("fixed", toks, {})], raw))]
    # distance 32768 (rows repeat every 128 rows of 256 bytes), lengths 258 through codes 285 and 284 + 31
    base = rng.integers(0, 256, (128, 255), dtype=np.uint8)
    build, raw = _grey(255, 400, np.concatenate([base] * 4)[:400])
    for via in (False, True):
        toks = _tokenize(raw, 32768, via284=via)
        assert any(isinstance(t, tuple) and t[1] == 32768 for t in toks)
        files.append(build(_stream([("dynamic", toks, {})], raw)))
        files.append(build(_stream([("fixed", toks, {})], raw)))
    # distance 1 runs through a one-code distance tree
    build, raw = _grey(300, 20, np.repeat(rng.integers(0, 256, (20, 1), dtype=np.uint8), 300, axis=1))
    toks = _tokenize(raw, 1)
    files.append(build(_stream([("dynamic", toks, {"dist_lens": [1]})], raw)))
    # literals only: an empty distance tree; and 15-bit codes (a code of lengths 1, 2, ..., 14, 15, 15)
    build, raw = _grey(16, 9, rng.integers(1, 15, (9, 16), dtype=np.uint8))
    toks = list(raw)
    files.append(build(_stream([("dynamic", toks, {"dist_lens": [0]})], raw)))
    lit = [0] * 286
    for s, l in zip(list(range(15)) + [256], list(range(1, 15)) + [15, 15]):
        lit[s] = l
    files.append(build(_stream([("dynamic", toks, {"lit_lens": lit, "dist_lens": [0]})], raw)))
    # windows referenced across block boundaries
    build, raw = _grey(100, 200, np.concatenate([rng.integers(0, 256, (10, 100), dtype=np.uint8)] * 20))
    toks = _tokenize(raw, 1010)
    files.append(build(_stream([("dynamic" if k % 2 else "fixed", toks[k:k + 40], {}) for k in range(0, len(toks), 40)], raw)))
    for f in files:
        assert not isinstance(pil_read(f), Exception)
    st = check_batch(files)
    assert (st[:, 3] > 0).all()


def _damaged():
    """(name, file) pairs of damaged streams; the good image every batch also holds is first."""
    rng = np.random.default_rng(5)
    w, h = 40, 30
    rows = random_rows(rng, w, h, 2, 8, "photo")
    raw = filter_rows(rows, 3, (0, 1, 2, 3, 4))
    row = 1 + 3 * w
    z = zlib.compress(raw)

    def bad_adler(s):
        return s[:-1] + bytes([s[-1] ^ 1])

    def sync(data):
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        return co.compress(data) + co.flush(zlib.Z_SYNC_FLUSH)
    out = [("good", png_file(w, h, 2, 8, z)),
           ("short on a row boundary", png_file(w, h, 2, 8, zlib.compress(raw[:5 * row]))),
           ("short mid-row", png_file(w, h, 2, 8, zlib.compress(raw[:5 * row + 7]))),
           ("empty image data", png_file(w, h, 2, 8, zlib.compress(b""))),
           ("cut stream", png_file(w, h, 2, 8, z[:-6])),
           ("cut stream mid-row", png_file(w, h, 2, 8, z[:len(z) // 2])),
           ("no final block, 5 rows", png_file(w, h, 2, 8, b"\x78\x9c" + sync(raw[:5 * row]))),
           ("full stream minus 8 bytes", png_file(w, h, 2, 8, z[:-8])),
           ("exact, bad Adler", png_file(w, h, 2, 8, bad_adler(z))),
           ("longer, bad Adler", png_file(w, h, 2, 8, bad_adler(zlib.compress(raw + bytes(50))))),
           ("short, bad Adler", png_file(w, h, 2, 8, bad_adler(zlib.compress(raw[:5 * row])))),
           ("invalid block after image", png_file(w, h, 2, 8, b"\x78\x9c" + sync(raw) + b"\x07\xff\xff\xff")),
           ("stops after a non-final block", png_file(w, h, 2, 8, b"\x78\x9c" + sync(raw))),
           ("filter byte 5", png_file(w, h, 2, 8, zlib.compress(raw[:3 * row] + b"\x05" + raw[3 * row + 1:]))),
           ("bad IDAT CRC", bytearray(png_file(w, h, 2, 8, z)))]
    d = out[-1][1]
    p = d.index(b"IDAT")
    d[p + 4 + int.from_bytes(d[p - 4:p], "big")] ^= 1
    out[-1] = (out[-1][0], bytes(d))
    # a match reaching before the stream, right at the start and after the image's last byte
    wr = D.BitWriter()
    D.fixed(wr, [7, (3, 5)] + list(raw[4:]), True)
    out.append(("distance too far", png_file(w, h, 2, 8, D.zlib_wrap(wr.getvalue(), raw))))
    wr = D.BitWriter()
    D.fixed(wr, list(raw) + [(3, len(raw) + 1)], True)
    out.append(("distance too far after the image", png_file(w, h, 2, 8, D.zlib_wrap(wr.getvalue(), raw))))
    wr = D.BitWriter()
    D.fixed(wr, list(raw) + [(3, len(raw))], True)
    out.append(("valid match after the image", png_file(w, h, 2, 8, D.zlib_wrap(wr.getvalue(), raw))))
    # single-byte corruptions anywhere in the stream
    for k in range(40):
        s = bytearray(z)
        s[int(rng.integers(2, len(s)))] ^= int(rng.integers(1, 256))
        out.append((f"corrupt byte {k}", png_file(w, h, 2, 8, bytes(s))))
    return out


def test_damaged_streams_follow_pil():
    cases = _damaged()
    outcome = {n: not isinstance(pil_read(f), Exception) for n, f in cases}
    # the rule the decoder restates, as PIL shows it
    assert outcome["short on a row boundary"] and not outcome["short mid-row"] and outcome["longer, bad Adler"]
    assert not outcome["exact, bad Adler"] and not outcome["invalid block after image"] and outcome["stops after a non-final block"]
    assert not outcome["filter byte 5"] and outcome["bad IDAT CRC"]
    assert not outcome["empty image data"] and not outcome["no final block, 5 rows"] and outcome["cut stream"]
    files = [f for _, f in cases]
    st = check_batch(files)
    assert st[0, 0] == 0
    with pytest.raises(Exception, match="corrupt PNG data"):
        preprocess.decode_png_batch([files[0], cases[2][1]])


def test_status_counts_chunks_and_serial_bytes():
    """A default stream of dynamic blocks over several chunks is decoded by confirmed chunks; a Z_FIXED stream has no block header
    the search can find, so chunk 0 decodes all of it serially; a damaged stream falls back to the serial decoder."""
    rng = np.random.default_rng(2)
    h, w = 720, 1280
    raw = h * (1 + w * 3)
    default = pil_png(photo(h, w, 5))
    fixed = make_png(rng, w, h, 2, 8, "photo", types=(1,), strategy=zlib.Z_FIXED)
    damaged = bytearray(default)
    damaged[len(damaged) // 2] ^= 0x55
    files = [default, fixed, bytes(damaged)]
    _, st = preprocess.decode_png_batch(files, with_status=True)
    chunks = -(-len(default) // 65536)
    assert st[0, 0] == 0 and chunks - 1 <= st[0, 1] <= chunks and st[0, 1] > 2, st[0]
    assert st[0, 2] == st[0, 1] - 1 and 0 < st[0, 3] < raw // 2, st[0]
    assert st[1, 0] == 0 and st[1, 1] > 2 and st[1, 2] == 0 and st[1, 3] == raw, st[1]
    check_batch(files)


def _mixed(rng):
    from jpeg_cases import photo as ph
    import io as _io
    from PIL import Image

    def jpeg(im):
        b = _io.BytesIO()
        Image.fromarray(im).save(b, "JPEG", quality=90)
        return b.getvalue()
    host_png = png_file(33, 21, 0, 16, zlib.compress(filter_rows(random_rows(rng, 33, 21, 0, 16), 2, (0, 1))))
    return [jpeg(ph(200, 300, 1)), pil_png(ph(240, 320, 2)), make_png(rng, 77, 51, 3, 4, "photo"), host_png,
            make_png(rng, 300, 200, 6, 16, "photo"), ph(100, 150, 3)]


@pytest.mark.parametrize("lanes", [None, 2])
@pytest.mark.parametrize("extra", ["plain", "tiling", "rendering"])
def test_mixed_batches_through_submit_images(golden_weights, voc_anchors, lanes, extra):
    rng = np.random.default_rng(4)
    items = _mixed(rng)
    assert [preprocess.png_gpu_decodable(x) if isinstance(x, bytes) else None for x in items] == [False, True, True, False, True, None]
    ref_items = [pil_read(x) if isinstance(x, bytes) else x for x in items]
    batches = [items[:4], items[2:], [items[1], items[4], items[0]]]
    refs = [ref_items[:4], ref_items[2:], [ref_items[1], ref_items[4], ref_items[0]]]

    def make():
        if lanes is None:
            p = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 8, obj_thresh=0.7, iou_thresh=0.5)
            p.engine.set_weights(golden_weights)
        else:
            p = LanedPipeline(lanes, "yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 8, obj_thresh=0.7, iou_thresh=0.5, sm_split=False)
            p.set_weights(golden_weights)
        if extra == "tiling":
            p.enable_tiling(1, 1)
        if extra == "rendering":
            p.enable_rendering()
        return p
    pipe, ref = make(), make()
    pipe.enable_png_decode()

    def run(p, bs):
        out = []
        for b in bs:
            t = p.submit_images(b)
            out.append(DetectionPipeline.records(*p.collect(t)))
            if extra == "rendering":
                out.append(p.rendered(t))
        return out
    assert run(pipe, batches) == run(ref, refs)


def test_letterbox_batch_device_and_errors(golden_weights, voc_anchors):
    from oracle import preprocess_ref
    rng = np.random.default_rng(6)
    items = _mixed(rng)
    out = preprocess.letterbox_batch_device(items, IN_HW, gpu_png=True).cpu().numpy()
    for got, x in zip(out, items):
        np.testing.assert_array_equal(got, preprocess_ref.letterbox(pil_read(x) if isinstance(x, bytes) else x, IN_HW))
    victim = dict(_damaged())["short mid-row"]
    assert preprocess.png_gpu_decodable(victim)
    with pytest.raises(Exception, match="corrupt PNG data: image 1"):
        preprocess.letterbox_batch_device([items[1], victim], IN_HW, gpu_png=True)
    pipe = DetectionPipeline("yolo_mobilev1", IN_HW, voc_anchors, 20, 0.75, 4, obj_thresh=0.7, iou_thresh=0.5)
    pipe.engine.set_weights(golden_weights)
    pipe.enable_png_decode()
    t = pipe.submit_images([items[0], victim, items[1]])
    t2 = pipe.submit_images([items[1]])
    with pytest.raises(Exception, match="corrupt PNG data: image 1"):
        pipe.collect(t)
    pipe.collect(t2)


def test_serve_gpu_png_keeps_its_lines(tmp_path, golden_weights):
    import serve
    from k210_yolo_framework_b200.hdf5_write import save_keras_weights
    ckpt = tmp_path / "model.h5"
    save_keras_weights(str(ckpt), golden_weights)
    d = tmp_path / "imgs"
    d.mkdir()
    rng = np.random.default_rng(8)
    for i, x in enumerate(_mixed(rng)[:5]):
        (d / (f"{i}.jpg" if i == 0 else f"{i}.png")).write_bytes(x)
    (d / "dog.jpg").write_bytes(open(os.path.join(GOLDEN, "dog.jpg"), "rb").read())

    class A:
        pass
    a = A()
    a.ckpt, a.images, a.model_def, a.depth_multiplier, a.image_size, a.class_num = str(ckpt), str(d), "yolo_mobilev1", 0.75, (224, 320), 20
    a.anchors, a.batch, a.obj_thresh, a.iou_thresh, a.decode_threads = os.path.join(GOLDEN, "voc_anchor.npy"), 4, 0.7, 0.5, 2
    with open(tmp_path / "host.jsonl", "w") as fh:
        assert serve.serve(a, fh) == 6
    a.gpu_png = True
    with open(tmp_path / "gpu.jsonl", "w") as fh:
        assert serve.serve(a, fh) == 6
    assert open(tmp_path / "gpu.jsonl").read() == open(tmp_path / "host.jsonl").read()
    assert serve.load_image(str(d / "1.png")).shape == (240, 320, 3)
    assert isinstance(serve.load_image(str(d / "1.png"), gpu_png=True), bytes)
    assert [json.loads(l)["image"] for l in open(tmp_path / "gpu.jsonl").read().splitlines()][0] == str(d / "0.jpg")
