"""Many streams in one tracker: each stream of a ``streams=S`` tracker gives, bit for bit, what it gives tracked alone, for
SORT, ByteTrack and OC-SORT, whatever the mix of streams in the batches (against the oracles on small streams, against
the single-stream GPU tracker on 200 streams); ``reset(s)`` / ``reset_tracks(s)`` restart one stream only; bad stream
input is refused with nothing changed; several videos through one ``serve.py --track`` run, and ``evaluate_mot.py
--streams N``, give what each video or sequence gives alone."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bytetrack_streams
import ocsort_streams
from conftest import ROOT
from oracle import bytetrack_ref, ocsort_ref, sort_ref
from test_gpu_track import WORKER, _crowded, _equal, _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _frames(method, rng, C, K, n):
    """n seeded frames (boxes, counts, scores) of the tracker's test streams."""
    if method == "sort":
        return [(b, c, np.zeros((C, K), np.float32)) for b, c in _stream(rng, C, K, n)]
    if method == "bytetrack":
        return bytetrack_streams.stream(rng, C, K, n)
    return ocsort_streams.stream(rng, C, K, n)


def _crowded_frames(method, C, K, n):
    if method == "sort":
        return [(b, c, np.full((C, K), 0.9, np.float32)) for b, c in _crowded(C, K, n)]
    return (bytetrack_streams if method == "bytetrack" else ocsort_streams).crowded(C, K, n)


def _tracker(method, C, K, streams=1, **kw):
    from k210_yolo_framework_b200.track import ByteTracker, OcSortTracker, Tracker
    cls = {"sort": Tracker, "bytetrack": ByteTracker, "ocsort": OcSortTracker}[method]
    return cls(C, K, device=0, streams=streams, **kw)


def _oracle(method, C, K, **kw):
    if method == "sort":
        s = sort_ref.Sort(C, K, **kw)
        return lambda p, b, c, sc: s.update(p, b, c)
    t = (bytetrack_ref.ByteTrack if method == "bytetrack" else ocsort_ref.OcSort)(C, K, **kw)
    return t.update


def _launch(tracker, batch, C, K, rng=None):
    """One launch over `batch`, a list of (stream, position, frame), each frame in a random row of the block (rows not in
    batch order); returns ids [n, C, K] and boxes [n, C, K, 4] in batch order."""
    from k210_yolo_framework_b200.dist import DetectionGather
    n = len(batch)
    rows = (rng.permutation(2 * n + 1)[:n] if rng is not None else np.arange(n)).astype(np.int32)
    buf = torch.zeros((2 * n + 1, C * (K * 6 + 1)), dtype=torch.int32)
    dets, counts = DetectionGather.split(buf, C, K)
    for r, (_, _, (b, c, s)) in zip(rows, batch):
        dets[r, :, :, :4] = torch.from_numpy(b.view(np.int32))
        dets[r, :, :, 4] = torch.from_numpy(s.view(np.int32))
        counts[r] = torch.from_numpy(c)
    dets, counts = DetectionGather.split(buf.to(DEV), C, K)
    pos, strm, last = tracker_check(tracker, batch)
    p = torch.tensor(pos, dtype=torch.int64, device=DEV)
    st = torch.tensor(strm, dtype=torch.int32, device=DEV)
    io_ = torch.full((n, C, K), 7, dtype=torch.int32, device=DEV)
    bo = torch.full((n, C, K, 4), 7.0, dtype=torch.float32, device=DEV)
    tracker.update(dets, counts, torch.from_numpy(rows).to(DEV), p, n, io_, bo, torch.cuda.current_stream(), last, st)
    return io_.cpu().numpy(), bo.cpu().numpy()


def tracker_check(tracker, batch):
    from k210_yolo_framework_b200.track import check_positions
    return check_positions([p for _, p, _ in batch], [s for s, _, _ in batch], tracker.last_positions)


def _mix(rng, streams, hold_back=0):
    """The frames of `streams` (lists of (position, frame)) merged in a random order that keeps each stream's order, cut into
    batches of 1..9; stream `hold_back` sits out from its fourth frame until every other stream has ended, then comes back."""
    queues = [list(s) for s in streams]
    held = queues[hold_back][3:] if len(streams) > 1 else []
    if held:
        queues[hold_back] = queues[hold_back][:3]
    order = []
    while any(queues):
        live = [i for i, q in enumerate(queues) if q]
        i = live[int(rng.integers(0, len(live)))]
        order.append((i,) + queues[i].pop(0))
        if held and not any(queues):
            queues[hold_back], held = held, []
    batches, a = [], 0
    while a < len(order):
        m = int(rng.integers(1, 10))
        batches.append(order[a:a + m])
        a += m
    return batches


def _run_mixed(tracker, batches, C, K, rng):
    """Each stream's (ids, boxes) per frame, in its frame order."""
    out = {}
    for batch in batches:
        ids, boxes = _launch(tracker, batch, C, K, rng)
        for j, (s, _, _) in enumerate(batch):
            out.setdefault(s, ([], []))
            out[s][0].append(ids[j])
            out[s][1].append(boxes[j])
    return {s: (np.stack(a), np.stack(b)) for s, (a, b) in out.items()}


def _positions(rng, n, start):
    """n increasing positions from `start`, with gaps of 2 and one long gap."""
    pos, p = [], start
    for f in range(n):
        pos.append(p)
        p += 1 + (1 if rng.random() < 0.15 else 0) + (40 if f == n // 2 else 0)
    return pos


SETTINGS = {"sort": dict(max_age=3, min_hits=1), "bytetrack": dict(track_buffer=4), "ocsort": dict(max_age=5)}


@pytest.mark.parametrize("method", ["sort", "bytetrack", "ocsort"])
@pytest.mark.parametrize("S", [1, 3, 7])
def test_each_stream_equals_its_oracle_in_any_mix(method, S):
    C, K = 4, 12
    rng = np.random.default_rng(100 + S)
    streams, refs = [], []
    for s in range(S):
        n = 16 + 4 * s                                   # streams of different lengths, at very different positions
        frames = _frames(method, np.random.default_rng(1000 * S + s), C, K, n)
        pos = _positions(rng, n, 500 * (S - 1 - s))
        streams.append(list(zip(pos, frames)))
        o = _oracle(method, C, K, **SETTINGS[method])
        out = [o(p, *f) for p, f in zip(pos, frames)]
        refs.append((np.stack([r[0] for r in out]), np.stack([r[1] for r in out])))
    assert all((r[0] >= 0).sum() > 5 for r in refs)
    for trial in range(2):
        batches = _mix(rng, streams, hold_back=trial % S)
        t = _tracker(method, C, K, S, **SETTINGS[method])
        got = _run_mixed(t, [[(s, p, f) for s, p, f in b] for b in batches], C, K, rng)
        for s in range(S):
            _equal(*got[s], *refs[s], f"{method} stream {s} of {S}, trial {trial}")


@pytest.mark.parametrize("method", ["sort", "bytetrack", "ocsort"])
def test_200_streams_equal_the_single_stream_tracker(method):
    """More CTAs than SMs, one stream with a class at its track bound among light ones; every stream against the
    single-stream GPU tracker on the same frames and batches."""
    C, K, S, n = 20, 30, 200, 12
    crowd = 7
    kw = {"sort": dict(max_age=9), "bytetrack": dict(track_buffer=30), "ocsort": dict(max_age=30)}[method]
    streams = []
    for s in range(S):
        frames = _crowded_frames(method, C, K, n) if s == crowd else _frames(method, np.random.default_rng(s), C, K, n)
        streams.append([(3 * s + f, fr) for f, fr in enumerate(frames)])
    rng = np.random.default_rng(5)
    # each stream's frames in two launches, split at a stream-dependent frame, the launches mixing every stream
    cut = [1 + s % (n - 1) for s in range(S)]
    batches = [[(s, p, fr) for s in range(S) for p, fr in streams[s][:cut[s]]],
               [(s, p, fr) for s in range(S) for p, fr in streams[s][cut[s]:]]]
    for b in batches:                               # round after round of one frame per stream, streams in random order
        key = {id(x): (x[1] - 3 * x[0], rng.random()) for x in b}
        b.sort(key=lambda x: key[id(x)])
    t = _tracker(method, C, K, S, **kw)
    got = _run_mixed(t, batches, C, K, rng)
    one = _tracker(method, C, K, 1, **kw)
    for s in range(S):
        one.reset()
        ids, boxes = [], []
        for part in (streams[s][:cut[s]], streams[s][cut[s]:]):
            i, b = _launch(one, [(0, p, fr) for p, fr in part], C, K)
            ids.append(i)
            boxes.append(b)
        _equal(*got[s], np.concatenate(ids), np.concatenate(boxes), f"{method} stream {s}")
    assert (got[crowd][0][:, 0] >= 0).sum() > 0


@pytest.mark.parametrize("method", ["sort", "bytetrack", "ocsort"])
def test_reset_of_one_stream(method):
    C, K, S, n = 4, 12, 3, 16
    frames = [_frames(method, np.random.default_rng(70 + s), C, K, n) for s in range(S)]
    t = _tracker(method, C, K, S, **SETTINGS[method])
    first = [[(s, 100 * s + f, frames[s][f]) for s in range(S)] for f in range(n // 2)]
    _run_mixed(t, first, C, K, np.random.default_rng(0))
    t.reset(1, torch.cuda.current_stream())
    assert t.last_positions[1] is None and t.last_positions[0] is not None
    second = [[(s, (0 if s == 1 else 100 * s) + f, frames[s][f]) for s in range(S)] for f in range(n // 2, n)]
    got = _run_mixed(t, second, C, K, np.random.default_rng(1))
    for s in range(S):
        o = _oracle(method, C, K, **SETTINGS[method])
        pos = [(0 if s == 1 else 100 * s) + f for f in range(n)]
        out = [o(p, *fr) for p, fr in zip(pos, frames[s])]
        if s == 1:          # restarted: ids from 1 and frame count 0, as a fresh stream over the second half
            o = _oracle(method, C, K, **SETTINGS[method])
            out = [o(p, *fr) for p, fr in zip(pos[n // 2:], frames[s][n // 2:])]
        else:
            out = out[n // 2:]
        _equal(*got[s], np.stack([r[0] for r in out]), np.stack([r[1] for r in out]), f"{method} stream {s}")
    assert got[1][0].max() >= 1 and got[1][0][got[1][0] > 0].min() == 1


def test_out_of_range_streams_get_cleared_outputs_and_touch_no_state():
    """The C entry point, below the Python checks: a frame of stream -1 or S gets id -1 and box 0, and the other frames run
    as without it."""
    from k210_yolo_framework_b200._lib import check
    C, K, S = 4, 12, 2
    frames = _frames("sort", np.random.default_rng(3), C, K, 3)
    good = _tracker("sort", C, K, S)
    ref = _launch(good, [(0, 0, frames[0]), (1, 0, frames[1])], C, K)
    t = _tracker("sort", C, K, S)
    from k210_yolo_framework_b200.dist import DetectionGather
    buf = torch.zeros((4, C * (K * 6 + 1)), dtype=torch.int32)
    dets, counts = DetectionGather.split(buf, C, K)
    for r, (b, c, _) in enumerate([frames[2], frames[0], frames[2], frames[1]]):
        dets[r, :, :, :4] = torch.from_numpy(b.view(np.int32))
        counts[r] = torch.from_numpy(c)
    dets, counts = DetectionGather.split(buf.to(DEV), C, K)
    rows = torch.arange(4, dtype=torch.int32, device=DEV)
    pos = torch.zeros(4, dtype=torch.int64, device=DEV)
    strm = torch.tensor([-1, 0, S, 1], dtype=torch.int32, device=DEV)
    io_ = torch.full((4, C, K), 7, dtype=torch.int32, device=DEV)
    bo = torch.full((4, C, K, 4), 7.0, dtype=torch.float32, device=DEV)
    from k210_yolo_framework_b200._lib import lib
    check(lib.k2y_track_update_streams(t.state.data_ptr(), S, t.stride, dets.data_ptr(), counts.data_ptr(), dets.stride(0),
                                       rows.data_ptr(), pos.data_ptr(), strm.data_ptr(), 4, C, K, 1, 3, 0.3, io_.data_ptr(),
                                       bo.data_ptr(), torch.cuda.current_stream().cuda_stream))
    ids, boxes = io_.cpu().numpy(), bo.cpu().numpy()
    for j in (0, 2):
        assert (ids[j] == -1).all() and (boxes[j] == 0).all()
    _equal(ids[[1, 3]], boxes[[1, 3]], *ref, "in-range frames")
    assert torch.equal(t.state, good.state)
    # a stride below one stream's state is refused, nothing launched
    from k210_yolo_framework_b200._lib import K2YError
    with pytest.raises(K2YError):
        check(lib.k2y_track_update_streams(t.state.data_ptr(), S, t.stride - 256, dets.data_ptr(), counts.data_ptr(),
                                           dets.stride(0), rows.data_ptr(), pos.data_ptr(), strm.data_ptr(), 4, C, K, 1, 3, 0.3,
                                           io_.data_ptr(), bo.data_ptr(), torch.cuda.current_stream().cuda_stream))


# ---------------------------------------------------------------------------------------------------------------------
# DetectionPipeline, serve.py and evaluate_mot.py
# ---------------------------------------------------------------------------------------------------------------------
def _videos(tmp_path, lengths):
    """Motion-JPEG AVIs of the test scene, one per length, each shifted differently."""
    from test_gpu_video import _scene
    from test_video import _pil, build_avi, strip_dht
    out = []
    for v, n in enumerate(lengths):
        frames = [strip_dht(_pil(_scene(k + 5 * v), quality=90, subsampling=1)) for k in range(n)]
        p = tmp_path / f"cam{v}.avi"
        p.write_bytes(build_avi(frames, w=320, h=240, scale=1001, rate=30000))
        out.append(p)
    return out


def _pipe(tmp_path, streams=3, **kw):
    import serve
    from test_gpu_video import _args
    a = _args(tmp_path, tmp_path, 4)
    pipe, _, _ = serve.open_pipeline(a)
    pipe.enable_tracking(streams=streams, **kw)
    return pipe


def test_pipeline_refuses_bad_streams_and_stays_as_it_was(tmp_path):
    pipe = _pipe(tmp_path)
    img = np.full((240, 320, 3), 90, np.uint8)
    t = pipe.submit_images([img, img], frames=[0, 0], streams=[0, 2])
    pipe.collect(t)
    before = list(pipe._track["tracker"].last_positions)
    for kw in (dict(frames=[1, 1], streams=[0, 3]),          # stream out of range
               dict(frames=[1, 1], streams=[-1, 0]),
               dict(frames=[1, 1]),                          # streams missing with 3 streams
               dict(frames=[0, 1], streams=[0, 1]),          # position 0 does not follow stream 0's 0
               dict(frames=[2, 2], streams=[1, 1])):         # not increasing within stream 1
        with pytest.raises(ValueError):
            pipe.submit_images([img, img], **kw)
        assert pipe._track["tracker"].last_positions == before
    with pytest.raises(ValueError):
        pipe.submit_images([img], streams=[0])               # streams without frames
    t = pipe.submit_images([img, img, img], frames=[1, 1, 0], streams=[0, 2, 1])   # the same positions on other streams
    pipe.collect(t)
    ids, _ = pipe.tracks(t)
    assert ids.shape[0] == 3
    pipe.reset_tracks(2)
    assert pipe._track["tracker"].last_positions == [1, 0, None]
    t = pipe.submit_images([img], frames=[0], streams=[2])
    pipe.collect(t)


def _serve_lines(args):
    from test_gpu_video import _serve
    return _serve(args)[1]


@pytest.mark.parametrize("tracker", ["sort", "bytetrack", "ocsort"])
def test_serve_several_videos_equals_each_alone(tmp_path, tracker):
    from test_gpu_video import _args
    vids = _videos(tmp_path, [9, 5, 7] if tracker != "bytetrack" else [6, 8])
    kw = dict(track=True, tracker=tracker)
    together = [json.loads(l) for l in _serve_lines(_many_args(tmp_path, vids, **kw))]
    for v in vids:
        alone = [json.loads(l) for l in _serve_lines(_args(tmp_path, v, 4, **kw))]
        mine = [l for l in together if l["video"] == str(v)]
        assert mine == alone, v
    assert sum(d.get("track") is not None for l in together for d in l["detections"]) > 3
    assert [l["video"] for l in together[:len(vids)]] == [str(v) for v in vids]    # interleaved, one frame each in turn


def _many_args(tmp_path, vids, **kw):
    from test_gpu_video import _args
    a = _args(tmp_path, vids[0], 4, **kw)
    a.images = [str(v) for v in vids]
    return a


def test_serve_several_videos_draws_each_avi_as_alone(tmp_path):
    from test_gpu_video import _args
    vids = _videos(tmp_path, [7, 4, 5])
    out_all = tmp_path / "all"
    _serve_lines(_many_args(tmp_path, vids, track=True, draw=str(out_all)))
    plain = [json.loads(l) for l in _serve_lines(_many_args(tmp_path, vids))]
    for v in vids:
        one = tmp_path / f"one_{v.stem}"
        _serve_lines(_args(tmp_path, v, 4, track=True, draw=str(one)))
        assert (out_all / f"{v.stem}.avi").read_bytes() == (one / f"{v.stem}.avi").read_bytes()
        alone = [json.loads(l) for l in _serve_lines(_args(tmp_path, v, 4))]
        assert [l for l in plain if l["video"] == str(v)] == alone     # without --track: detected in shared batches


def test_two_gpus_track_several_videos_as_one(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    vids = _videos(tmp_path, [7, 5, 6])
    a = _many_args(tmp_path, vids, track=True)
    one = _serve_lines(a)
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    argv = [a.ckpt] + [str(v) for v in vids] + ["--anchors", a.anchors, "--batch", "4", "--obj_thresh", "0.3", "--track"]
    env = dict(os.environ, K2Y_ROOT=ROOT, PYTHONPATH=ROOT, K2Y_OUT=str(tmp_path / "two.jsonl"))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29551", str(script)] + argv, capture_output=True, text=True, timeout=540, env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert open(tmp_path / "two.jsonl").read().splitlines() == one


def test_evaluate_mot_streams_equal_the_sequential_run(tmp_path):
    import evaluate_mot
    from test_gpu_mot import _args, _mot_sequence
    for name, L in (("PEOPLE-01", 9), ("PEOPLE-02", 4), ("PEOPLE-03", 7), ("PEOPLE-04", 2)):
        _mot_sequence(tmp_path / "train", name, L)
    res, files = {}, {}
    for n in (1, 3):
        out = tmp_path / f"res{n}"
        res[n] = evaluate_mot.evaluate(_args(tmp_path, [tmp_path / "train"], results=out, streams=n))
        files[n] = {f: (out / f).read_bytes() for f in sorted(os.listdir(out))}
    assert res[1] == res[3]
    assert files[1] == files[3] and len(files[1]) == 4
    assert all(len(v) > 0 for v in files[1].values())
