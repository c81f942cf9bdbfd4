"""Tracking on the GPU: SORT (``k2y_track_update``, csrc/track.cu; oracle/sort_ref.py states the rules), ByteTrack
(``k2y_bytetrack_update``, csrc/bytetrack.cu; oracle/bytetrack_ref.py) and OC-SORT (``k2y_ocsort_update``, csrc/ocsort.cu;
oracle/ocsort_ref.py).  ``Tracker``, ``ByteTracker`` and ``OcSortTracker`` each own the device state of `streams`
independent streams (1 by default) and run one launch per batch of frames over a gathered record block, one CTA per stream
(the ``*_update_streams`` entry points); a batch may mix the streams' frames.  Each stream's ids count from 1, so a track
is identified by (stream, id)."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import torch

from ._lib import check, lib

MAX_TRACKS_PER_CLASS = 1024
BYTETRACK_MAX_TRACKS_PER_CLASS = 4096
OCSORT_MAX_TRACKS_PER_CLASS = 4096
OCSORT_MAX_DELTA_T = 8


def _whole(name: str, v, lo: int = 0, hi: Optional[int] = None, unit: str = "") -> None:
    """Raises ValueError unless v is a whole number (not a bool) in lo..hi."""
    if isinstance(v, bool) or int(v) != v or v < lo or (hi is not None and v > hi):
        raise ValueError(f"{name} {v}: a whole number{unit} " + (f"in {lo}..{hi}" if hi is not None else f">= {lo}"))


def _unit(name: str, v) -> None:
    if not 0.0 <= float(v) <= 1.0:
        raise ValueError(f"{name} {v} is outside [0, 1]")


def check_setting(K: int, max_age, min_hits, iou_thresh) -> None:
    """Raises ValueError for a setting the tracker does not take (oracle/sort_ref.py ``check_setting``)."""
    _whole("max_age", max_age, unit=" of frames")
    _whole("min_hits", min_hits)
    _unit("iou_thresh", iou_thresh)
    if K * (int(max_age) + 1) > MAX_TRACKS_PER_CLASS:
        raise ValueError(f"max_per_class {K} x (max_age {max_age} + 1) tracks per class exceed the {MAX_TRACKS_PER_CLASS} the "
                         f"tracker holds: max_age <= {MAX_TRACKS_PER_CLASS // K - 1} at max_per_class {K}")


def check_positions(positions: Sequence[int], streams: Optional[Sequence[int]], last: Sequence[Optional[int]]):
    """(positions, streams, {stream: its last position in the batch}) of a batch of frames, as ints, for a tracker of
    len(last) streams whose last positions so far are `last` (None: the stream has not started).  `streams` gives each
    frame's stream (None: every frame is stream 0).  Raises ValueError for a stream outside 0..len(last) - 1, a negative
    position, or a position that does not increase along its stream; the streams are independent of one another."""
    pos = [int(p) for p in positions]
    strm = [0] * len(pos) if streams is None else [int(s) for s in streams]
    if len(strm) != len(pos):
        raise ValueError(f"{len(strm)} streams for {len(pos)} frame positions")
    seen = {}
    for p, s in zip(pos, strm):
        if not 0 <= s < len(last):
            raise ValueError(f"stream {s} is outside 0..{len(last) - 1}")
        prev = seen.get(s, last[s])
        if p < 0 or (prev is not None and p <= prev):
            raise ValueError(f"frame position {p} of stream {s} does not follow {prev}: positions increase along a stream, "
                             "from 0")
        seen[s] = p
    return pos, strm, seen


class _StreamTracker:
    """The device state of `streams` streams and their launches, for the tracker whose C entry points are `state_bytes`
    and `update` (an ``*_update_streams``): each takes (C, K) and then `state_args` or `setting`.  The states lie
    state_bytes apart."""

    def __init__(self, C: int, K: int, state_bytes, state_args: tuple, update, setting: tuple, device, streams: int = 1):
        _whole("streams", streams, 1)
        self.C, self.K, self.streams = int(C), int(K), int(streams)
        self._update, self._setting = update, setting
        nbytes = ctypes.c_size_t()
        check(state_bytes(self.C, self.K, *state_args, ctypes.byref(nbytes)))
        self.stride = nbytes.value
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.state = torch.zeros(self.streams * self.stride, dtype=torch.uint8, device=dev)
        self.last_positions: List[Optional[int]] = [None] * self.streams    # host copy, to refuse positions that do not increase

    def reset(self, stream: Optional[int] = None, cuda_stream: Optional[torch.cuda.Stream] = None) -> None:
        """Starts every stream anew (`stream` None), or stream `stream` alone; enqueued on `cuda_stream` (default: the
        current one)."""
        if stream is not None:
            _whole("stream", stream, 0, self.streams - 1)
        state = self.state if stream is None else self.state[int(stream) * self.stride:(int(stream) + 1) * self.stride]
        with torch.cuda.stream(cuda_stream or torch.cuda.current_stream(self.state.device)):
            state.zero_()
        if stream is None:
            self.last_positions = [None] * self.streams
        else:
            self.last_positions[int(stream)] = None

    def check_positions(self, positions: Sequence[int], streams: Optional[Sequence[int]] = None) -> list:
        """The positions as ints; raises ValueError unless they increase along each stream, from that stream's last one on
        (``check_positions`` of the module)."""
        return check_positions(positions, streams, self.last_positions)[0]

    def update(self, dets: torch.Tensor, counts: torch.Tensor, rows: torch.Tensor, positions: torch.Tensor, n_frames: int,
               ids_out: torch.Tensor, boxes_out: torch.Tensor, stream: torch.cuda.Stream, last_position,
               streams_of_frames: Optional[torch.Tensor] = None) -> None:
        """Frames rows[:n_frames] of the block (dets [N, C, K, 6] int32 and counts [N, C] of one buffer, same row stride), at
        positions[:n_frames] (device int64, checked with ``check_positions``), of the streams streams_of_frames[:n_frames]
        (device int32; None: every frame is stream 0); writes ids_out [>= n_frames, C, K] int32 and boxes_out [>= n_frames,
        C, K, 4] float32.  `last_position`: the batch's last position (one stream), or {stream: its last position in the
        batch} as ``check_positions`` gives it."""
        if dets.stride(0) != counts.stride(0):
            raise ValueError("dets and counts must share their row stride (a gather block)")
        if streams_of_frames is not None and (streams_of_frames.dtype != torch.int32 or streams_of_frames.device != self.state.device):
            raise ValueError("streams_of_frames must be int32 on the tracker's device")
        check(self._update(self.state.data_ptr(), self.streams, self.stride, dets.data_ptr(), counts.data_ptr(), dets.stride(0),
                           rows.data_ptr(), positions.data_ptr(),
                           None if streams_of_frames is None else streams_of_frames.data_ptr(), int(n_frames), self.C, self.K,
                           *self._setting, ids_out.data_ptr(), boxes_out.data_ptr(), ctypes.c_void_p(stream.cuda_stream)))
        last = last_position if isinstance(last_position, dict) else {0: last_position}
        for s, p in last.items():
            self.last_positions[int(s)] = int(p)


class Tracker(_StreamTracker):
    """SORT tracks over `C` classes of at most `K` records per frame, of `streams` independent streams.  ``update``
    enqueues one launch for a batch of frames; ``reset`` starts every stream, or one, anew.  Both are asynchronous on the
    CUDA stream given and must be ordered among themselves."""
    def __init__(self, C: int, K: int, max_age: int = 1, min_hits: int = 3, iou_thresh: float = 0.3, device=None,
                 streams: int = 1):
        check_setting(K, max_age, min_hits, iou_thresh)
        self.max_age, self.min_hits, self.iou_thresh = int(max_age), int(min_hits), float(iou_thresh)
        super().__init__(C, K, lib.k2y_track_state_bytes, (self.max_age,), lib.k2y_track_update_streams,
                         (self.max_age, self.min_hits, self.iou_thresh), device, streams)


def check_bytetrack_setting(K: int, track_thresh, match_thresh, track_buffer) -> None:
    """Raises ValueError for a ByteTrack setting the tracker does not take: a class holds K (max(track_buffer, 1) + 2)
    tracks within a frame (oracle/bytetrack_ref.py ``max_tracks``), at most 4096."""
    _unit("track_thresh", track_thresh)
    _unit("match_thresh", match_thresh)
    _whole("track_buffer", track_buffer, unit=" of frames")
    cap = BYTETRACK_MAX_TRACKS_PER_CLASS
    if K * (max(int(track_buffer), 1) + 2) > cap:
        raise ValueError(f"max_per_class {K} x (max(track_buffer {track_buffer}, 1) + 2) tracks per class exceed the {cap} the "
                         f"tracker holds: track_buffer <= {cap // K - 2} at max_per_class {K}")


class ByteTracker(_StreamTracker):
    """``Tracker``'s interface over ByteTrack: the tracks of `streams` streams over `C` classes of at most `K` records per
    frame, the score in word 4 of each record."""
    def __init__(self, C: int, K: int, track_thresh: float = 0.5, match_thresh: float = 0.8, track_buffer: int = 30,
                 fuse_score: bool = True, device=None, streams: int = 1):
        check_bytetrack_setting(K, track_thresh, match_thresh, track_buffer)
        self.track_thresh, self.match_thresh = float(track_thresh), float(match_thresh)
        self.track_buffer, self.fuse_score = int(track_buffer), bool(fuse_score)
        super().__init__(C, K, lib.k2y_bytetrack_state_bytes, (self.track_buffer,), lib.k2y_bytetrack_update_streams,
                         (self.track_thresh, self.match_thresh, self.track_buffer, int(self.fuse_score)), device, streams)


def check_ocsort_setting(K: int, det_thresh, max_age, min_hits, iou_thresh, delta_t, inertia) -> None:
    """Raises ValueError for an OC-SORT setting the tracker does not take: a class holds K (max_age + 1) tracks
    (oracle/ocsort_ref.py ``max_tracks``), at most 4096, and each track a ring of delta_t observations, delta_t <= 8."""
    _whole("max_age", max_age, unit=" of frames")
    _whole("min_hits", min_hits)
    for name, v in (("iou_thresh", iou_thresh), ("det_thresh", det_thresh), ("inertia", inertia)):
        _unit(name, v)
    _whole("delta_t", delta_t, 1, OCSORT_MAX_DELTA_T, unit=" of frames")
    cap = OCSORT_MAX_TRACKS_PER_CLASS
    if K * (int(max_age) + 1) > cap:
        raise ValueError(f"max_per_class {K} x (max_age {max_age} + 1) tracks per class exceed the {cap} the OC-SORT tracker "
                         f"holds: max_age <= {cap // K - 1} at max_per_class {K}")


class OcSortTracker(_StreamTracker):
    """``Tracker``'s interface over OC-SORT: the tracks of `streams` streams over `C` classes of at most `K` records per
    frame, the score in word 4 of each record."""
    def __init__(self, C: int, K: int, det_thresh: float = 0.6, max_age: int = 30, min_hits: int = 3, iou_thresh: float = 0.3,
                 delta_t: int = 3, inertia: float = 0.2, use_byte: bool = False, device=None, streams: int = 1):
        check_ocsort_setting(K, det_thresh, max_age, min_hits, iou_thresh, delta_t, inertia)
        self.det_thresh, self.max_age, self.min_hits = float(det_thresh), int(max_age), int(min_hits)
        self.iou_thresh, self.delta_t, self.inertia, self.use_byte = float(iou_thresh), int(delta_t), float(inertia), bool(use_byte)
        super().__init__(C, K, lib.k2y_ocsort_state_bytes, (self.max_age, self.delta_t), lib.k2y_ocsort_update_streams,
                         (self.det_thresh, self.max_age, self.min_hits, self.iou_thresh, self.delta_t, self.inertia,
                          int(self.use_byte)), device, streams)
