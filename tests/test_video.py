"""Video input and output without a GPU: the standard Huffman tables the baseline parser gives DHT-less files, the Motion-JPEG AVI
reader (cv2-written files, hand-built files of every index kind, dropped frames, JUNK and LIST rec chunks, OpenDML, padded and
two-field frames), AviWriter read back by the reader and by OpenCV's FFmpeg backend, and serve.py's content sniffing."""
import io
import os
import struct

import numpy as np
import pytest

from k210_yolo_framework_b200 import preprocess, video
from oracle import jpeg_ref


def _img(h=48, w=64, seed=0):
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(seed)
    base = np.stack([(xx * 3 + yy * (c + 1) + 40 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 10, base.shape), 0, 255).astype(np.uint8)


def _pil(img, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", **kw)
    return b.getvalue()


def _segments(data):
    """(marker, start, end) of every marker segment before the SOS, and the SOS's offset."""
    out, i = [], 2
    while data[i + 1] != 0xDA:
        n = int.from_bytes(data[i + 2:i + 4], "big")
        out.append((data[i + 1], i, i + 2 + n))
        i += 2 + n
    return out, i


def strip_dht(data, keep=()):
    """The file without its DHT segments, except tables (class, id) in `keep` (each DHT rewritten with the kept ones)."""
    segs, sos = _segments(data)
    out = bytearray(data[:2])
    for m, a, b in segs:
        if m != 0xC4:
            out += data[a:b]
            continue
        body, k, kept = data[a + 4:b], 0, b""
        while k < len(body):
            n = 17 + sum(body[k + 1:k + 17])
            if (body[k] >> 4, body[k] & 15) in keep:
                kept += body[k:k + n]
            k += n
        if kept:
            out += b"\xff\xc4" + struct.pack(">H", 2 + len(kept)) + kept
    return bytes(out + data[sos:])


def dht_tables(data):
    """{(class, id): (bits[1..16], values)} of every DHT table in a file."""
    segs, _ = _segments(data)
    out = {}
    for m, a, b in segs:
        if m == 0xC4:
            body, k = data[a + 4:b], 0
            while k < len(body):
                bits = list(body[k + 1:k + 17])
                out[(body[k] >> 4, body[k] & 15)] = (bits, list(body[k + 17:k + 17 + sum(bits)]))
                k += 17 + sum(bits)
    return out


LAYOUTS = {"444": dict(subsampling=0), "422": dict(subsampling=1), "420": dict(subsampling=2)}


@pytest.mark.parametrize("quality", [50, 90, 100])
def test_pil_writes_the_annex_k3_tables(quality):
    """PIL (libjpeg-turbo) with optimize=False writes T.81 Annex K.3's tables: the tables the parser now uses for a slot 0 or 1
    no DHT defines."""
    tabs = dht_tables(_pil(_img(), quality=quality, subsampling=1))
    assert tabs == {(0, 0): jpeg_ref.STD_DC_LUMA, (1, 0): jpeg_ref.STD_AC_LUMA,
                    (0, 1): jpeg_ref.STD_DC_CHROMA, (1, 1): jpeg_ref.STD_AC_CHROMA}


def _huff_section(data):
    """The derived Huffman tables k2y_jpeg_plan writes into the blob for one file (the blob's last 1424 bytes per table)."""
    buf = np.frombuffer(data, np.uint8)
    n = preprocess._jpeg_plan([buf], np.zeros(1, np.int64), np.zeros(1, np.int64), None)
    blob = np.zeros(n + 16, np.uint8)
    blob = blob[(-blob.ctypes.data) % 16:][:n]
    preprocess._jpeg_plan([buf], np.zeros(1, np.int64), np.zeros(1, np.int64), blob)
    tables = 2 * (1 if _pil_mode(data) == "L" else 3)
    return blob[n - tables * 1424:].copy()


def _pil_mode(data):
    from PIL import Image
    return Image.open(io.BytesIO(data)).mode


@pytest.mark.parametrize("layout", ["444", "422", "420", "gray"])
def test_default_tables_equal_the_dht_tables_pil_writes(layout):
    """A DHT-less file plans exactly the derived tables of the same file with PIL's DHT segments: the default tables are PIL's,
    through the same derivation and the same blob."""
    img = _img(40, 72)
    from PIL import Image
    data = _pil(np.asarray(Image.fromarray(img).convert("L")), quality=85) if layout == "gray" else _pil(img, quality=85, **LAYOUTS[layout])
    bare = strip_dht(data)
    assert len(bare) < len(data) and not dht_tables(bare)
    assert preprocess.inspect_jpeg(bare)[2:] == (True, "")
    np.testing.assert_array_equal(_huff_section(bare), _huff_section(data))


@pytest.mark.parametrize("keep", [[(0, 0)], [(1, 1)], [(0, 0), (1, 0)], [(0, 1), (1, 1)], [(0, 0), (1, 0), (0, 1)]])
def test_files_with_some_tables_left_out_are_gpu_decodable(keep):
    data = _pil(_img(), quality=75, subsampling=2)
    part = strip_dht(data, keep)
    assert sorted(dht_tables(part)) == sorted(keep)
    assert preprocess.inspect_jpeg(part)[2:] == (True, "")
    assert preprocess.gpu_decodable(part)
    np.testing.assert_array_equal(_huff_section(part), _huff_section(data))


def test_an_undefined_slot_2_keeps_the_old_reason():
    """libjpeg-turbo's std_huff_tables fills slots 0 and 1 only: a scan naming an undefined table 2 stays with PIL."""
    data = bytearray(strip_dht(_pil(_img(), quality=75, subsampling=2)))
    _, sos = _segments(bytes(data))
    assert data[sos + 4] == 3
    data[sos + 8] = 0x22            # component 2 selects DC / AC tables 2
    assert preprocess.inspect_jpeg(bytes(data))[2:] == (False, "Huffman table not defined before the scan")
    data[sos + 8] = 0x02            # AC table 2 only
    assert preprocess.inspect_jpeg(bytes(data))[2:] == (False, "Huffman table not defined before the scan")


def test_progressive_files_without_dht_are_not_changed():
    data = _pil(_img(), quality=75, progressive=True)
    assert preprocess.inspect_jpeg(data)[2] is False
    assert preprocess.inspect_jpeg_progressive(strip_dht(data))[2] is False


# ---------------------------------------------------------------------------------------------------------------------
# Hand-built AVI files
# ---------------------------------------------------------------------------------------------------------------------
def chunk(cid, data):
    return cid + struct.pack("<I", len(data)) + data + (b"\0" if len(data) & 1 else b"")


def lst(kind, *parts):
    return chunk(b"LIST", kind + b"".join(parts))


def strl(kind, handler, w, h, scale, rate, n, comp=None):
    strh = struct.pack("<4s4sIHHIIIIIIIIhhhh", kind, handler, 0, 0, 0, 0, scale, rate, 0, n, 0, 0xFFFFFFFF, 0, 0, 0, w, h)
    strf = struct.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, comp or handler, w * h * 3, 0, 0, 0, 0) if kind == b"vids" else bytes(18)
    return lst(b"strl", chunk(b"strh", strh), chunk(b"strf", strf))


def build_avi(frames, w=64, h=48, scale=1, rate=25, micro=40000, index="movi", junk=False, rec=False, audio=False,
              handler=b"MJPG", comp=None):
    """An AVI with `frames` (bytes; b"" is a dropped frame) as its video stream: `index` "movi" (idx1 offsets from the movi
    fourcc), "absolute", or None; `junk` puts JUNK chunks in the header and between frames, `rec` groups frames in LIST rec,
    `audio` puts an audio stream in front (the video is stream 01, with audio chunks between its frames)."""
    vid = b"01dc" if audio else b"00dc"
    streams = ([strl(b"auds", b"\0\0\0\0", 0, 0, 1, 8000, 0)] if audio else []) + [strl(b"vids", handler, w, h, scale, rate, len(frames), comp)]
    avih = struct.pack("<IIIIIIIIII16x", micro, 0, 0, 0x10, len(frames), 0, len(streams), 0, w, h)
    hdrl = lst(b"hdrl", chunk(b"avih", avih), *streams)
    pre = hdrl + (chunk(b"JUNK", bytes(37)) if junk else b"")
    body, entries = b"", []
    for k, fr in enumerate(frames):
        part = b""
        if junk and k % 2:
            part += chunk(b"JUNK", bytes(k + 1))
        if audio:
            part += chunk(b"00wb", bytes(10))
        at = len(body) + len(part)
        part += chunk(vid, fr)
        if rec:
            part = lst(b"rec ", part)
            at += 12
        entries.append((at, len(fr)))
        body += part
    movi_fourcc = 12 + len(pre) + 8
    idx = b""
    if index:
        base = 4 if index == "movi" else movi_fourcc + 4
        idx = chunk(b"idx1", b"".join(struct.pack("<4sIII", vid, 0x10, base + at, n) for at, n in entries))
    riff = b"AVI " + pre + lst(b"movi", body) + idx
    return b"RIFF" + struct.pack("<I", len(riff)) + riff


def _frames(n=5, **kw):
    return [_pil(_img(seed=k), quality=60 + 5 * k, **kw) for k in range(n)]


def _write(tmp_path, data, name="v.avi"):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


@pytest.mark.parametrize("index", ["movi", "absolute", None])
@pytest.mark.parametrize("junk,rec,audio", [(False, False, False), (True, False, False), (False, True, False), (True, True, True)])
def test_reader_finds_every_frame(tmp_path, index, junk, rec, audio):
    frames = _frames()
    v = video.open_video(_write(tmp_path, build_avi(frames, index=index, junk=junk, rec=rec, audio=audio)))
    assert isinstance(v, video.MjpegAvi)
    assert (v.n_frames, v.fps, v.frame_hw, v.codec) == (5, 25.0, (48, 64), "MJPG")
    assert [v.frame_bytes(k) for k in range(5)] == frames == list(v.frames())
    assert [v.time(k) for k in range(5)] == [k / 25 for k in range(5)]


def test_reader_uses_the_compression_code_and_avih_rate(tmp_path):
    frames = _frames(3)
    v = video.open_video(_write(tmp_path, build_avi(frames, rate=0, micro=33367, handler=b"\0\0\0\0", comp=b"AVRn")))
    assert isinstance(v, video.MjpegAvi) and v.codec == "AVRn"
    assert v.fps == pytest.approx(1e6 / 33367) and v.time(2) == pytest.approx(2 * 0.033367)
    v = video.open_video(_write(tmp_path, build_avi(frames, scale=1001, rate=30000, handler=b"dmb1"), "w.avi"))
    assert v.codec == "dmb1" and v.time(2) == 2 * 1001 / 30000


@pytest.mark.parametrize("index", ["movi", None])
def test_dropped_frames_keep_their_positions(tmp_path, index):
    frames = _frames(4)
    stored = [frames[0], b"", frames[1], frames[2], b"", b"", frames[3]]
    v = video.open_video(_write(tmp_path, build_avi(stored, index=index)))
    assert v.n_frames == 4
    assert [v.frame_bytes(k) for k in range(4)] == frames
    assert [v.position(k) for k in range(4)] == [0, 2, 3, 6]
    assert [v.time(k) for k in range(4)] == [0.0, 2 / 25, 3 / 25, 6 / 25]


def test_a_broken_index_falls_back_to_the_movi_walk(tmp_path):
    frames = _frames(3)
    data = bytearray(build_avi(frames, index="movi"))
    at = data.rindex(b"idx1") + 8
    data[at + 8:at + 12] = struct.pack("<I", 12345)       # the first entry points nowhere
    v = video.open_video(_write(tmp_path, bytes(data)))
    assert [v.frame_bytes(k) for k in range(3)] == frames


def test_padded_and_two_field_frames_are_cut_at_the_first_eoi(tmp_path):
    a, b = _frames(2)
    rst = _pil(_img(seed=3), quality=70, restart_marker_blocks=1)
    stored = [a + bytes(7), a + b, rst + b"\xff\xd9" + bytes(3), a + b"\xff" * 5, b + b"\x00\xff\xd8junk"]
    v = video.open_video(_write(tmp_path, build_avi(stored)))
    assert [v.frame_bytes(k) for k in range(5)] == [a, a, rst, a, b]
    assert [v.payload(k) for k in range(5)] == stored
    assert video.cut_frame(a[:-2]) == a[:-2]                # no complete image: kept as stored
    assert video.jpeg_end(b"not a jpeg") is None


def test_non_mjpeg_avi_goes_to_ffmpeg(tmp_path):
    cv2 = pytest.importorskip("cv2")
    p = str(tmp_path / "x.avi")
    w = cv2.VideoWriter(p, cv2.CAP_FFMPEG, cv2.VideoWriter_fourcc(*"mp4v"), 10.0, (64, 48))
    assert w.isOpened()
    for k in range(4):
        w.write(_img(seed=k))
    w.release()
    v = video.open_video(p)
    assert isinstance(v, video.FfmpegVideo) and v.n_frames == 4 and v.fps == 10.0 and v.frame_hw == (48, 64)
    cap = cv2.VideoCapture(p, cv2.CAP_FFMPEG)
    for k, got in enumerate(v.frames()):
        ok, bgr = cap.read()
        np.testing.assert_array_equal(got, bgr[..., ::-1])
    # frames asked for out of order and frames another rank keeps
    load = v.loader(keep=lambda k: k % 2 == 1)
    assert load(3).shape == (48, 64, 3) and load(1).shape == (48, 64, 3)
    with pytest.raises(ValueError, match="after the stream passed it"):
        load(0)


def _packets(path):
    import cv2
    cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
    cap.set(cv2.CAP_PROP_FORMAT, -1)
    n, fps = int(cap.get(cv2.CAP_PROP_FRAME_COUNT)), cap.get(cv2.CAP_PROP_FPS)
    out = []
    while True:
        ok, pkt = cap.read()
        if not ok:
            break
        out.append(pkt.tobytes())
    return n, fps, out


@pytest.mark.parametrize("api", ["CAP_OPENCV_MJPEG", "CAP_FFMPEG"])
def test_reader_reads_cv2_mjpeg_avis(tmp_path, api):
    cv2 = pytest.importorskip("cv2")
    p = str(tmp_path / "cv.avi")
    w = cv2.VideoWriter(p, getattr(cv2, api), cv2.VideoWriter_fourcc(*"MJPG"), 12.0, (64, 48))
    assert w.isOpened()
    for k in range(7):
        w.write(_img(seed=k))
    w.release()
    v = video.open_video(p)
    n, fps, pkts = _packets(p)
    assert isinstance(v, video.MjpegAvi) and (v.n_frames, v.fps, v.frame_hw) == (n, fps, (48, 64)) == (7, 12.0, (48, 64))
    assert [v.payload(k) for k in range(7)] == pkts
    for k in range(7):
        assert pkts[k].startswith(v.frame_bytes(k)) and v.frame_bytes(k).endswith(b"\xff\xd9")


@pytest.mark.parametrize("limit", [None, 20000, 6000])
def test_avi_writer_reads_back_through_the_reader_and_ffmpeg(tmp_path, limit):
    pytest.importorskip("cv2")
    frames = _frames(12) + [_pil(_img(seed=99), quality=95) + b"\0"]        # an odd size: the chunk gets its pad byte
    p = str(tmp_path / "w.avi")
    kw = {} if limit is None else {"riff_limit": limit}
    with video.AviWriter(p, 30000 / 1001, (48, 64), **kw) as w:
        for f in frames:
            w.write(f)
    data = open(p, "rb").read()
    riffs = data.count(b"AVIX")
    assert (riffs > 0) == (limit is not None) and (b"indx" in data) == (limit is not None)
    if limit == 6000:
        assert riffs >= 3
    v = video.open_video(p)
    assert isinstance(v, video.MjpegAvi) and v.n_frames == 13 and v.fps == 30000 / 1001 and v.frame_hw == (48, 64)
    assert [v.payload(k) for k in range(13)] == frames
    n, fps, pkts = _packets(p)
    assert (n, pkts) == (13, frames) and fps == pytest.approx(30000 / 1001)
    if limit is not None:       # the frames of the AVIX RIFFs are reached through the super index
        assert v._entries[-1][1] > data.index(b"AVIX")


def test_avi_writer_refuses_a_frame_of_another_size(tmp_path):
    p = str(tmp_path / "w.avi")
    with video.AviWriter(p, 25, (48, 64)) as w:
        w.write(_pil(_img()))
        with pytest.raises(ValueError, match="frame 1 is 65x48"):
            w.write(_pil(_img(48, 65)))
        w.write(_pil(_img(seed=2)))
    assert video.open_video(p).n_frames == 2


def test_serve_sniffs_videos_by_content(tmp_path):
    import serve
    d = tmp_path / "imgs"
    d.mkdir()
    (d / "a.jpg").write_bytes(_pil(_img()))
    (d / "clip.avi").write_bytes(build_avi(_frames(2)))
    (d / "clip.mp4").write_bytes(b"\0\0\0\x18ftypisom" + bytes(16))
    lst_file = tmp_path / "list.txt"
    lst_file.write_text(f"{d / 'a.jpg'}\n")
    assert not serve.is_video(str(d)) and not serve.is_video(str(lst_file))
    assert serve.list_images(str(d)) == [str(d / "a.jpg")]            # videos in a directory are not picked up
    assert serve.list_images(str(lst_file)) == [str(d / "a.jpg")]
    assert serve.is_video(str(d / "clip.avi")) and serve.is_video(str(d / "clip.mp4"))
    mkv = tmp_path / "x.bin"
    mkv.write_bytes(b"\x1a\x45\xdf\xa3" + bytes(20))
    assert serve.is_video(str(mkv))
    txt = tmp_path / "RIFF.txt"
    txt.write_text("RIFF is not a video\n")
    assert not serve.is_video(str(txt))
