"""The GPU trackers (SORT, ByteTrack, OC-SORT) against their oracles bit for bit where kernels go wrong: every decision of
tests/tracker_edges.py exactly on its threshold and one step to either side, tie-heavy frames, and the size bounds (class_num
1 to 1024, a class at exactly its track capacity, two crowded classes on one warp)."""
import numpy as np
import pytest
import torch

import bytetrack_streams
import ocsort_streams
from test_gpu_bytetrack import _run
from test_gpu_track import _equal
from tracker_edges import EDGE_STREAMS, boundary_cases, run_ref, variant

pytestmark = pytest.mark.gpu

CASES = boundary_cases()


def _tracker(kind, C, K, kw):
    from k210_yolo_framework_b200.track import ByteTracker, OcSortTracker, Tracker
    return {"sort": Tracker, "bytetrack": ByteTracker, "ocsort": OcSortTracker}[kind](C, K, device=0, **kw)


def _check(kind, C, K, kw, frames, positions, splits, what):
    ref = run_ref(kind, C, K, kw, frames, positions)
    for split in splits:
        got = _run(_tracker(kind, C, K, kw), frames, positions, split, C, K, torch.device("cuda", 0))
        _equal(*got, *ref, f"{what}, batches of {split}")
    return ref


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_thresholds_at_and_beside_the_boundary(case):
    ran = 0
    for side in (-1, 0, 1):
        v = variant(case, side)
        if v is None:
            continue
        kw, frames = v
        _check(case.tracker, case.C, case.K, kw, frames, case.positions, (1, len(frames)), f"{case.name} side {side}")
        ran += 1
    assert ran >= (1 if case.kind == "const" else 2)


@pytest.mark.parametrize("name,kind,kw,make", EDGE_STREAMS, ids=[e[0] for e in EDGE_STREAMS])
def test_edge_streams(name, kind, kw, make):
    frames = make(2, 64)
    _check(kind, 2, 64, kw, frames, list(range(len(frames))), (1, 7, len(frames)), name)


# -- size bounds -------------------------------------------------------------------------------------------------------------
def _sparse_stream(rng, C, K, n_frames, classes):
    """Frames in which only `classes` have records: a few moving, overlapping objects each, scores in both bands."""
    out = []
    objs = {c: [(rng.random(2) * 400, rng.normal(size=2) * 4, 10 + rng.random(2) * 40) for _ in range(min(K, 3))]
            for c in classes}
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for c, os_ in objs.items():
            recs = [(p + v * f + rng.normal(size=2), wh) for p, v, wh in os_ if rng.random() < 0.9][:K]
            for k, (p, wh) in enumerate(recs):
                boxes[c, k] = [p[1], p[0], p[1] + wh[1], p[0] + wh[0]]
                scores[c, k] = rng.choice([0.9, 0.75, 0.3, 0.6])
            counts[c] = len(recs)
        out.append((boxes, counts, scores))
    return out


SETTINGS = {"sort": dict(max_age=2, min_hits=1), "bytetrack": dict(track_buffer=3), "ocsort": dict(max_age=3, min_hits=1)}


@pytest.mark.parametrize("kind", ["sort", "bytetrack", "ocsort"])
@pytest.mark.parametrize("C", [1, 9, 1024])
def test_class_num_1_9_and_1024(kind, C):
    rng = np.random.default_rng(C)
    classes = sorted({0, C - 1} | set(rng.integers(0, C, min(C, 12)).tolist()))
    frames = _sparse_stream(rng, C, 4, 12, classes)
    ref = _check(kind, C, 4, SETTINGS[kind], frames, list(range(12)), (1, 12), f"{kind} C {C}")
    assert (ref[0] >= 0).sum() > 10


@pytest.mark.parametrize("kw", [dict(max_age=0, min_hits=0), dict(max_age=3, min_hits=1)])
def test_sort_one_record_per_class(kw):
    frames = _sparse_stream(np.random.default_rng(5), 6, 1, 20, [0, 2, 5])
    _check("sort", 6, 1, kw, frames, list(range(20)), (1, 20), f"sort K 1 {kw}")


def _fill(C, K, n_frames, classes, period=1):
    """K new boxes in each of `classes` every `period` frames, overlapping nothing of before (SORT and OC-SORT keep each
    until max_age removes it, ByteTrack confirms it in the next frame and then loses it)."""
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for n, c in enumerate(classes):
            for i in range(K):
                y, x = 40.0 * i, 100.0 + 40.0 * (f // period) + 15.0 * n
                boxes[c, i] = [y, x, y + 10, x + 10]
                scores[c, i] = 0.9
            counts[c] = K
        out.append((boxes, counts, scores))
    return out


@pytest.mark.parametrize("K,max_age", [(32, 31), (128, 7)])
def test_sort_a_class_of_exactly_1024_tracks(K, max_age):
    from oracle import sort_ref
    frames = _fill(2, K, max_age + 4, [0])
    s = sort_ref.Sort(2, K, max_age=max_age)
    live = 0
    for p, (b, c, _) in enumerate(frames):
        s.update(p, b, c)
        live = max(live, len(s.tracks[0]))
    assert live == 1024
    _check("sort", 2, K, dict(max_age=max_age), frames, list(range(len(frames))), (5,), f"sort {K} x {max_age + 1}")


def test_bytetrack_at_4096_tracks_per_class():
    from oracle import bytetrack_ref
    C, K, B = 2, 128, 30
    assert bytetrack_ref.max_tracks(K, B) == 4096
    frames = bytetrack_streams.crowded(C, K, B + 6)
    ref = _check("bytetrack", C, K, dict(track_buffer=B), frames, list(range(len(frames))), (16,), "bytetrack 4096")
    assert (ref[0] >= 0).sum() > K * (B // 2)     # K (B / 2 + 2) tracks alive at the end (the bound is not tight)


def test_ocsort_a_class_of_exactly_4096_tracks():
    from oracle import ocsort_ref
    C, K, A = 2, 128, 31
    frames = ocsort_streams.crowded(C, K, A + 3)
    t = ocsort_ref.OcSort(C, K, max_age=A)
    ref, live = [], 0
    for p, f in enumerate(frames):
        ref.append(t.update(p, *f))
        live = max(live, len(t.tracks[0]))
    assert live == 4096
    got = _run(_tracker("ocsort", C, K, dict(max_age=A)), frames, list(range(len(frames))), 16, C, K, torch.device("cuda", 0))
    _equal(*got, np.stack([r[0] for r in ref]), np.stack([r[1] for r in ref]), "ocsort 4096")


@pytest.mark.parametrize("kind,kw,period", [("bytetrack", dict(track_buffer=2), 2), ("ocsort", dict(max_age=2, min_hits=0), 1)])
def test_two_crowded_classes_on_one_warp(kind, kw, period):
    """Classes 3 and 11 share a warp (8 warps stride over the classes): the births of both, and of class 5 between them,
    take their ids in class order every frame."""
    frames = _fill(16, 64, 8, [3, 5, 11], period)
    ref = _check(kind, 16, 64, kw, frames, list(range(8)), (1, 3, 8), f"{kind} classes 3 and 11")
    assert (ref[0][:, 11] >= 0).sum() > 64 and (ref[0][:, 3] >= 0).sum() > 64
