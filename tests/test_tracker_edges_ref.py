"""The boundary cases of tests/tracker_edges.py really are on their boundary: the quantity equals the threshold exactly
(computed with the oracle's own helpers), and the oracle's ids or boxes at the threshold differ from those one step past
it on the side that flips.  A case that does not flip would let a kernel with > written as >= pass."""
import math

import numpy as np
import pytest

from oracle import bytetrack_ref, ocsort_ref, sort_ref
from tracker_edges import EDGE_STREAMS, boundary_cases, neighbour, run_ref, variant

CASES = boundary_cases()
MODULES = {"sort": sort_ref, "bytetrack": bytetrack_ref, "ocsort": ocsort_ref}


def _differ(a, b):
    return not (np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32)))


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_the_quantity_meets_the_threshold_exactly(case):
    if case.kind == "score":
        # a float32 score widened to float64 against a float64 bound: the case's score is the float32 at or just
        # above the bound, the one below it is under it
        below = float(np.nextafter(np.float32(case.quantity), np.float32(-math.inf)))
        assert case.quantity >= case.t > below
    else:
        assert case.quantity == case.t


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_the_outcome_flips_one_step_past_the_threshold(case, monkeypatch):
    at = run_ref(case.tracker, case.C, case.K, case.kw, case.frames, case.positions)
    if case.kind == "const":
        monkeypatch.setattr(MODULES[case.tracker], case.param, neighbour(case.t, case.flip))
        past = run_ref(case.tracker, case.C, case.K, case.kw, case.frames, case.positions)
    elif case.kind == "param" and isinstance(case.t, float) and not 0.0 <= neighbour(case.t, case.flip) <= 1.0:
        # past the setting's range (iou_thresh 0 or 1): the oracle takes it, the tracker's API does not
        past = run_ref(case.tracker, case.C, case.K, dict(case.kw, **{case.param: neighbour(case.t, case.flip)}),
                       case.frames, case.positions)
    else:
        kw, frames = variant(case, case.flip)
        past = run_ref(case.tracker, case.C, case.K, kw, frames, case.positions)
    assert _differ(at, past), f"{case.name}: the oracle gives the same ids and boxes one step past the threshold"


def test_bytetrack_duplicate_cost_cannot_be_0_15_exactly():
    """Why tests/tracker_edges.py has no case at the duplicate threshold: 1 - x for x in [0.5, 1] is exact, and 1 - 0.15
    is not a double."""
    x = 1.0 - bytetrack_ref.DUPLICATE_THRESH
    for v in (x, float(np.nextafter(x, 0)), float(np.nextafter(x, 1))):
        assert 1.0 - v != bytetrack_ref.DUPLICATE_THRESH


@pytest.mark.parametrize("name,tracker,kw,make", EDGE_STREAMS, ids=[e[0] for e in EDGE_STREAMS])
def test_edge_streams_track_something(name, tracker, kw, make):
    frames = make(2, 64)
    ids, _ = run_ref(tracker, 2, 64, kw, frames, list(range(len(frames))))
    assert (ids >= 0).sum() > 30
    assert len(set(ids[ids >= 0].tolist())) > 1
