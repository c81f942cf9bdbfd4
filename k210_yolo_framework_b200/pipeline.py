"""Batched detection pipeline: the whole hot path behind one call.

``DetectionPipeline.detect_host(x)`` is the user-facing end-to-end call for a batch of pre-processed images
held in (pinned) host memory: H2D copy -> network (one CUDA graph) -> decode + NMS -> [all-gather when the
job spans several GPUs] -> D2H of the fixed-size record blocks.  ``step_device()`` is the same work on inputs
already resident in HBM (what ``bench.py``'s ``value`` times).  ``submit``/``collect`` is the streaming form.
It is the batched form of keras_inference.py:87-135, which the reference runs for one image per process.

Streams: the network (one CUDA graph) runs on the caller's current stream; decode + NMS run on a second, high-priority
stream and read one of TWO head-buffer sets the network alternates between, so the decode of batch i overlaps the first
convolutions of batch i+1 (the small-grid layers leave SMs idle; the decode kernels are latency-bound).  With more than one
rank the all-gather (and the D2H copy of the gathered blocks) runs on a third stream into one of two gather buffers; H2D
copies use a fourth stream and land directly in one of two device input buffers the network is re-pointed at (one CUDA graph
per (input buffer, head set)), so there is no staging copy.  ``step_device(pipelined=False)`` (the default) makes the
caller's stream wait for the decode before returning — plain stream semantics; the streaming calls (``submit``/``collect``,
``step_device(pipelined=True)`` + ``wait_gathered()``) keep the overlap.

``submit_images`` takes raw host images of any size instead: each input slot has its own pinned staging buffer and its own
device ``image_hw`` [batch, 2]; the packed H2D copy and the batched letterbox (which also writes ``image_hw``) run on the copy
stream into the slot's uint8 input buffer, overlapping the previous batch's network, and the decode of that batch reads the
slot's ``image_hw``, so two batches in flight each carry their own original sizes.

``enable_rendering`` adds the drawn result to ``submit_images``: behind the NMS, on the decode stream, the batch's local records
are drawn onto its original images where they lie in the slot's device staging buffer and encoded as JPEG files;
``rendered(ticket)`` brings them back after ``collect`` with one exact-size copy.  The next ``submit_images`` into that input
slot waits for the render before it overwrites the originals.  ``enable_rendering(tracks=True)`` draws the batch's tracks
instead (``k2y_render_tracks``): behind the tracking launch, on the stream that runs it.

``enable_tiling`` makes ``submit_images`` detect on overlapping tiles of each image as well as on the whole image: a batch of
n <= batch // V images is letterboxed as n * V views, the network and the decode run on those, and one more per-class NMS
(``k2y_merge_views``, on the decode stream) merges each image's views into rows [0, n) of the gather slot, in image
coordinates and in the usual block format, so everything behind it is unchanged.  With ``tile_size`` each image gets its own
grid (``tiles.plan_grid``) and ``images_per_batch`` is the caller's; ``k2y_merge_views_ex`` then reads each image's view range
and the windows' interior sides from a table that travels in the batch's H2D copy, and can match by intersection over the
smaller box, fold the matched boxes into the kept one and drop records at the tiles' inner borders.

``enable_flip`` makes ``submit_images`` detect every view a second time, mirrored left to right (the flip the reference trains
with): the letterbox fetches the mirrored columns, and ``k2y_merge_views_mirror`` maps the mirrored views' records back into
the image while it loads them, then merges all views as above.  It combines with either grid, in either order.

``enable_tracking`` tracks objects across the frames of a stream, SORT-style (``track.Tracker``, oracle/sort_ref.py), with
ByteTrack (``track.ByteTracker``, oracle/bytetrack_ref.py) or with OC-SORT (``track.OcSortTracker``, oracle/ocsort_ref.py):
``submit_images(frames=...)`` gives each image's position in the stream, one ``k2y_track_update_streams``
(``k2y_bytetrack_update_streams``, ``k2y_ocsort_update_streams``) launch per batch runs behind the NMS / all-gather on the
stream that holds the gathered block, before its D2H, and ``tracks(ticket)`` returns each record's track id and box.  The
records are unchanged.  ``enable_tracking(streams=S)`` tracks S independent streams at once, one CTA each:
``submit_images(streams=...)`` names each frame's stream, and a batch may mix them.

``enable_png_decode`` makes ``submit_images`` decode the PNG files the GPU takes there too (``preprocess.png_gpu_decodable``),
in the same staging range and H2D copy as the batch's JPEGs; their status words travel beside the JPEGs'.
``enable_progressive_jpeg_decode`` does the same for progressive JPEGs (``preprocess.progressive_gpu_decodable``).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import ctypes

import numpy as np
import torch

from . import tiles, yolonet
from ._lib import check, lib
from .detect import DET_WORDS, KerasDetector
from .dist import DetectionGather
from .preprocess import BatchLayout, Staging, check_jpeg_status, check_png_status, check_progressive_status, letterbox_packed
from .track import check_positions

SLOTS = 2


def _check_merge_options(match, merge, border) -> None:
    if match not in tiles.MATCHES:
        raise ValueError(f"unknown match metric {match!r}: one of {', '.join(tiles.MATCHES)}")
    if merge not in tiles.MERGES:
        raise ValueError(f"unknown merge action {merge!r}: one of {', '.join(tiles.MERGES)}")
    if border is not None and not float(border) >= 0:
        raise ValueError(f"tile border {border}: at least 0 pixels")


class DetectionPipeline:
    def __init__(self, model_def: str, image_size: Sequence[int], anchors: np.ndarray, class_num: int, alpha: float,
                 batch: int, obj_thresh: float = 0.7, iou_thresh: float = 0.3, max_per_class: int = 30,
                 device: Optional[int] = None, world: int = 1, rank: int = 0, comm=None):
        self.batch, self.world, self.rank = int(batch), int(world), int(rank)
        self.in_hw = (int(image_size[0]), int(image_size[1]))
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        builder = getattr(yolonet, model_def)
        self.model, self.wrapper = builder([image_size[0], image_size[1], 3], len(anchors[0]), class_num, alpha=alpha,
                                           max_batch=batch, device=self.device_index)
        self.engine = self.model.engine
        out_hw = [(h, w) for h, w, _ in self.engine.out_shapes]
        self.detector = KerasDetector(anchors, image_size, out_hw, class_num, obj_thresh, iou_thresh, max_per_class,
                                      max_batch=batch, device=self.device_index)
        dev = torch.device("cuda", self.device_index)
        self.gather = DetectionGather(batch, class_num, max_per_class, dev, world=self.world, rank=self.rank, words=DET_WORDS,
                                      slots=SLOTS, comm=comm)
        self._img_hw = torch.tensor([[image_size[0], image_size[1]]] * batch, dtype=torch.float32, device=dev)
        self._side = torch.cuda.Stream(device=dev)          # all-gather + D2H of gathered blocks
        self._det_stream = torch.cuda.Stream(device=dev, priority=-1)   # decode + NMS (its CTAs go first when SM slots free up)
        self._head_sets = None                              # two sets of head buffers, created on first use
        self._heads_ready = [torch.cuda.Event() for _ in range(SLOTS)]   # network finished writing head set
        self._copy_stream = torch.cuda.Stream(device=dev)   # H2D
        self._host = [torch.empty(self.gather.bufs[0].shape, dtype=torch.int32).pin_memory() for _ in range(SLOTS)]
        self._in_f32: Optional[List[torch.Tensor]] = None   # device input buffers of the streaming API, created on first use
        self._in_u8: Optional[List[torch.Tensor]] = None
        self._h2d_done = [torch.cuda.Event() for _ in range(SLOTS)]
        self._in_free = [torch.cuda.Event() for _ in range(SLOTS)]       # network finished reading input slot
        self._det_done = [torch.cuda.Event() for _ in range(SLOTS)]      # local block of gather slot written
        self._gather_done = [torch.cuda.Event() for _ in range(SLOTS)]   # gather slot complete on this rank
        self._slot_free = [torch.cuda.Event() for _ in range(SLOTS)]     # last reader of gather slot is done
        self._d2h_done = [torch.cuda.Event() for _ in range(SLOTS)]
        # submit_images: per input slot a pinned staging buffer and the (h, w) of its images, created on first use
        self._staging: Optional[List[Staging]] = None
        self._slot_hw: Optional[List[torch.Tensor]] = None
        self._hw_free = [torch.cuda.Event() for _ in range(SLOTS)]       # decode finished reading the slot's image sizes
        self._rows: List[Optional[int]] = [None] * SLOTS                 # records collect returns per gather slot (None: all)
        # GPU-decoded JPEGs of the batch behind each gather slot: their batch positions and (pinned) status words
        self._jpeg_idx: List[list] = [[] for _ in range(SLOTS)]
        self._jpeg_status = [torch.zeros((batch, 4), dtype=torch.int32).pin_memory() for _ in range(SLOTS)]
        # enable_png_decode: the same for the batch's GPU-decoded PNGs
        self._gpu_png = False
        self._png_idx: List[list] = [[] for _ in range(SLOTS)]
        self._png_status = [torch.zeros((batch, 4), dtype=torch.int32).pin_memory() for _ in range(SLOTS)]
        # enable_progressive_jpeg_decode: the same for the batch's GPU-decoded progressive JPEGs
        self._gpu_progressive = False
        self._prog_idx: List[list] = [[] for _ in range(SLOTS)]
        self._prog_status = [torch.zeros((batch, 4), dtype=torch.int32).pin_memory() for _ in range(SLOTS)]
        self._steps = 0
        self._submitted = 0
        # enable_rendering: label atlas, colour table, quality, one encoder per gather slot (its files live until rendered())
        self._render = None
        self._render_done = [torch.cuda.Event() for _ in range(SLOTS)]   # files of gather slot ready to copy back
        self._render_free = [torch.cuda.Event() for _ in range(SLOTS)]   # render + encode finished with input slot's originals
        self._rendered_slot: List[bool] = [False] * SLOTS
        # enable_tiling / enable_flip: the grid and merge options asked for and the flip, from which tiles.plan_views derives
        # the rest: (rows, cols, overlap) or a tiles.SizedTiling, the most views of an image, images per batch, the merge's
        # options (None: k2y_merge_views), the per-view record block the decode writes and the merge reads (both on the decode
        # stream, so one block serves every batch) and per input slot the device (y0, x0) of its views
        self._grid = None
        self._merge_options = dict(match="iou", merge="suppress", match_thresh=None, border=None)
        self._flip = False
        self._tiling = None
        self._views = 1
        self._ipb = self.batch
        self._merge = None
        self._view_dets: Optional[torch.Tensor] = None
        self._view_counts: Optional[torch.Tensor] = None
        self._slot_yx: Optional[List[torch.Tensor]] = None
        # enable_tracking: the tracker, its pinned per-slot inputs and outputs and their device copies; per gather slot the
        # frames its batch tracked (None: not tracked)
        self._track = None
        self._track_n: List[Optional[int]] = [None] * SLOTS

    @property
    def images_per_batch(self) -> int:
        """Images one ``submit_images`` takes: ``batch``, ``batch // V`` with a rows x cols tiling, or the value given with
        ``tile_size``."""
        return self._ipb

    def enable_tiling(self, rows: Optional[int] = None, cols: Optional[int] = None, overlap: float = 0.2, *, tile_size=None,
                      images_per_batch: Optional[int] = None, match: str = "iou", merge: str = "suppress",
                      match_thresh: Optional[float] = None, border: Optional[float] = None) -> None:
        """From now on ``submit_images`` detects every image as V = 1 + rows * cols views: the whole image and rows x cols
        overlapping tiles of it (``tiles.tile_windows``), each letterboxed and decoded as the crop submitted as an image of
        its own would be.  A batch holds at most ``images_per_batch`` = batch // V images; their n * V views fill the input
        slot image-major, and ``k2y_merge_views`` merges each image's records behind the decode: boxes moved into image
        coordinates, ``index = view * nbox + index`` (``index // nbox`` tells the view), one more greedy NMS per class over
        the union.  ``collect`` returns the merged records in the usual format; rendering, the all-gather (rank r's images
        from row r * batch) and the flow control are unchanged.  Raises ``ValueError`` when V exceeds the batch or
        V * max_per_class exceeds what one merge holds (``k2y_merge_views_max_records``).

        ``tile_size=(th, tw)`` instead of rows and cols plans each image's grid from its own size (``tiles.plan_grid``): tiles
        of at most th x tw pixels, one view for an image that fits one tile, and at most ``max_views`` = min(batch //
        images_per_batch, k2y_merge_views_max_records() // max_per_class) views, so that a batch of `images_per_batch` images
        (required here, refused without tile_size) always fits.  Images' view ranges differ, and ``k2y_merge_views_ex`` merges
        them.  With either grid:
          `match`         "iou" (the default) or "ios": a candidate matches a kept record when their IoU, or their
                          intersection over the smaller box, exceeds `match_thresh` (default: the detector's iou_thresh);
          `merge`         "suppress" (the default) drops a matching candidate, "union" also grows the kept record's box to the
                          field-wise union of itself and the candidates it suppressed (score and index stay its own);
          `border`        None (the default) or m >= 0: a tile's record within m pixels of a tile edge that lies inside the
                          image is dropped before the merge (oracle/tiles_merge_ref.py states each rule exactly).
        With none of these set (and no ``enable_flip``), the merge is ``k2y_merge_views`` exactly.  With ``enable_flip``, before
        or after this call, every window is detected mirrored as well: V and max_views above count the mirrored views, and a
        tile_size grid is planned under max_views // 2.  Bad values raise ``ValueError`` and leave the pipeline as it was."""
        _check_merge_options(match, merge, border)
        if not 0 <= overlap < 1:
            raise ValueError(f"tile overlap {overlap} is outside [0, 1)")
        if tile_size is None:
            if rows is None or cols is None:
                raise ValueError("enable_tiling needs rows and cols, or tile_size")
            if images_per_batch is not None:
                raise ValueError("images_per_batch goes with tile_size; a rows x cols grid holds batch // (1 + rows * cols) images")
            rows, cols = int(rows), int(cols)
            if rows < 1 or cols < 1:
                raise ValueError(f"tiling {rows}x{cols}: at least one tile per axis")
            grid = ("grid", rows, cols, overlap)
        else:
            if rows is not None or cols is not None:
                raise ValueError("enable_tiling takes rows and cols, or tile_size, not both")
            if images_per_batch is None:
                raise ValueError("tile_size needs images_per_batch: the images one batch holds whatever their grids")
            th, tw = (int(v) for v in tile_size)
            if th < 1 or tw < 1:
                raise ValueError(f"tile size {th}x{tw}: at least one pixel per side")
            ipb = int(images_per_batch)
            if not 1 <= ipb <= self.batch:
                raise ValueError(f"images_per_batch {ipb} is outside 1..{self.batch}")
            grid = ("size", (th, tw), overlap, ipb)
        self._set_views(grid, dict(match=match, merge=merge, match_thresh=match_thresh, border=border), self._flip)

    def enable_flip(self, *, match: Optional[str] = None, merge: Optional[str] = None, match_thresh: Optional[float] = None,
                    border: Optional[float] = None) -> None:
        """From now on ``submit_images`` detects every view of an image a second time, mirrored left to right: the whole image
        then its mirror without tiling, or with W windows per image (``enable_tiling``, before or after this call) views 0 .. W-1
        as without flip and view W + v window v mirrored.  A mirrored view is letterboxed and decoded as ``np.fliplr`` of its
        crop submitted as an image of its own would be, and the merge maps its records back into the image
        (xmin = fl(fl(tw - xmax_m) + x0), xmax = fl(fl(tw - xmin_m) + x0); index = (W + v) * nbox + index) before merging every
        view as ``enable_tiling`` describes, with its options.  A batch holds batch // V images (V = 2, or 2 (1 + rows * cols));
        a tile_size grid plans its windows under max_views // 2.  `match`, `merge`, `match_thresh` and `border` are
        ``enable_tiling``'s merge options; each one not given keeps its value (from ``enable_tiling``, else the default), so the
        merge of a flip without tiling can take them too.  Raises ``ValueError`` when the views do not fit the batch or one
        merge, or for a bad option, and leaves the pipeline as it was."""
        given = dict(match=match, merge=merge, match_thresh=match_thresh, border=border)
        options = dict(self._merge_options, **{k: v for k, v in given.items() if v is not None})
        _check_merge_options(options["match"], options["merge"], options["border"])
        self._set_views(self._grid, options, True)

    def _set_views(self, grid, options: dict, flip: bool) -> None:
        """The one place the views follow from the grid, the merge options and the flip (``tiles.plan_views``); nothing changes
        when it raises."""
        tiling, V, ipb = tiles.plan_views(self.batch, self.gather.K, int(lib.k2y_merge_views_max_records()), grid, flip)
        legacy = not flip and grid[0] == "grid" and options == dict(match="iou", merge="suppress", match_thresh=None, border=None)
        dev = torch.device("cuda", self.device_index)
        self._grid, self._merge_options, self._flip = grid, options, flip
        self._tiling, self._views, self._ipb = tiling, V, ipb
        self._merge = None if legacy else dict(
            match=tiles.MATCHES.index(options["match"]), merge=tiles.MERGES.index(options["merge"]),
            thresh=float(self.detector.cfg.iou_thresh if options["match_thresh"] is None else options["match_thresh"]),
            border=None if options["border"] is None else float(options["border"]))
        self._nbox = sum(h * w for h, w in self.detector.out_hw) * self.detector.A      # boxes of one network input
        if self._view_dets is None:
            self._view_dets = torch.zeros((self.batch, self.gather.C, self.gather.K, DET_WORDS), dtype=torch.int32, device=dev)
            self._view_counts = torch.zeros((self.batch, self.gather.C), dtype=torch.int32, device=dev)
            self._slot_yx = [torch.zeros((self.batch, 2), dtype=torch.float32, device=dev) for _ in range(SLOTS)]

    def enable_tracking(self, max_age: Optional[int] = None, min_hits: Optional[int] = None, iou_thresh: Optional[float] = None, *,
                        method: str = "sort", track_thresh: float = 0.5, match_thresh: float = 0.8, track_buffer: int = 30,
                        fuse_score: bool = True, det_thresh: float = 0.6, delta_t: int = 3, inertia: float = 0.2,
                        use_byte: bool = False, streams: int = 1) -> None:
        """From now on ``submit_images`` takes `frames`, each image's position in a stream of frames, and tracks the objects of
        the stream as SORT does (oracle/sort_ref.py states every rule): per class, a Kalman filter per track, IoU association
        by optimal assignment, a track born for each unmatched detection and removed once it missed more than `max_age`
        frames (1 when left out), and reported once it was matched in `min_hits` frames in a row (3; or in the stream's first
        `min_hits` frames), matching at IoU `iou_thresh` (0.3).
        ``tracks(ticket)`` returns each record's id and track box.  A new call starts a new stream, as ``reset_tracks`` does.
        With `streams` S > 1 the pipeline tracks S independent streams (camera feeds, videos) in the same batches:
        ``submit_images`` then takes each frame's stream too, and each stream has its own tracks, frame count and ids from 1,
        exactly as if it were tracked alone, so a track is identified by (stream, id).  Each stream's state takes the
        tracker's ``k2y_*_state_bytes()`` on the device.
        Raises ``ValueError``, leaving the pipeline as it was, for a bad setting or when max_per_class * (max_age + 1)
        exceeds the 1024 tracks one class holds (max_age <= 33 at max_per_class 30, <= 9 at 100).

        ``method="bytetrack"`` tracks with ByteTrack instead (oracle/bytetrack_ref.py states every rule): a first association
        with the records scored above `track_thresh` (IoU times score with `fuse_score`, up to cost `match_thresh`), a second
        of the tracks left with the records scored in (0.1, track_thresh), births from records scored >= track_thresh + 0.1,
        and lost tracks kept `track_buffer` frames.  It only sees the records the detector keeps, so its second association
        needs an obj_thresh below track_thresh (0.1 as ByteTrack).  Each method refuses the other's arguments away from their
        defaults, and ByteTrack a setting where max_per_class * (max(track_buffer, 1) + 2) exceeds the 4096 tracks one
        class holds.

        ``method="ocsort"`` tracks with OC-SORT (oracle/ocsort_ref.py states every rule): SORT's filter, re-updated along a
        virtual path when a lost track is found again; a first association of the records scored above `det_thresh` by IoU
        plus `inertia` times the agreement of directions over `delta_t` frames; with `use_byte` a second of the tracks left
        with the records scored in (0.1, det_thresh) (it needs an obj_thresh below det_thresh); a third by the tracks' last
        observations.  It takes `max_age`, `min_hits` and `iou_thresh` too, with OC-SORT's defaults when left out (30, 3,
        0.3), refuses ByteTrack's arguments (and SORT and ByteTrack refuse its own away from their defaults), and refuses a
        setting where max_per_class * (max_age + 1) exceeds the 4096 tracks one class holds or delta_t is outside 1..8.  Its
        track box is the record's own box."""
        from .track import ByteTracker, OcSortTracker, Tracker
        sort_setting = (1 if max_age is None else max_age, 3 if min_hits is None else min_hits,
                        0.3 if iou_thresh is None else iou_thresh)
        sort_args = sort_setting != (1, 3, 0.3)
        byte_args = (track_thresh, match_thresh, track_buffer, fuse_score) != (0.5, 0.8, 30, True)
        oc_args = (det_thresh, delta_t, inertia, use_byte) != (0.6, 3, 0.2, False)
        if method == "sort":
            if byte_args:
                raise ValueError("track_thresh, match_thresh, track_buffer and fuse_score set ByteTrack: use method='bytetrack'")
            if oc_args:
                raise ValueError("det_thresh, delta_t, inertia and use_byte set OC-SORT: use method='ocsort'")
            tracker = Tracker(self.gather.C, self.gather.K, *sort_setting, self.device_index, streams)
        elif method == "bytetrack":
            if sort_args:
                raise ValueError("max_age, min_hits and iou_thresh set SORT: ByteTrack takes track_thresh, match_thresh, "
                                 "track_buffer and fuse_score")
            if oc_args:
                raise ValueError("det_thresh, delta_t, inertia and use_byte set OC-SORT: use method='ocsort'")
            tracker = ByteTracker(self.gather.C, self.gather.K, track_thresh, match_thresh, track_buffer, fuse_score,
                                  self.device_index, streams)
        elif method == "ocsort":
            if byte_args:
                raise ValueError("track_thresh, match_thresh, track_buffer and fuse_score set ByteTrack: OC-SORT takes max_age, "
                                 "min_hits, iou_thresh, det_thresh, delta_t, inertia and use_byte")
            tracker = OcSortTracker(self.gather.C, self.gather.K, det_thresh, 30 if max_age is None else max_age,
                                    3 if min_hits is None else min_hits, 0.3 if iou_thresh is None else iou_thresh, delta_t,
                                    inertia, use_byte, self.device_index, streams)
        else:
            raise ValueError(f"tracking method {method!r}: 'sort', 'bytetrack' or 'ocsort'")
        dev = torch.device("cuda", self.device_index)
        n, C, K = self.world * self.batch, self.gather.C, self.gather.K
        self._track = dict(
            tracker=tracker, rows=torch.empty(n, dtype=torch.int32, device=dev), pos=torch.empty(n, dtype=torch.int64, device=dev),
            streams=torch.empty(n, dtype=torch.int32, device=dev),
            streams_host=[torch.empty(n, dtype=torch.int32).pin_memory() for _ in range(SLOTS)],
            ids=torch.empty((n, C, K), dtype=torch.int32, device=dev), boxes=torch.empty((n, C, K, 4), dtype=torch.float32, device=dev),
            rows_host=[torch.empty(n, dtype=torch.int32).pin_memory() for _ in range(SLOTS)],
            pos_host=[torch.empty(n, dtype=torch.int64).pin_memory() for _ in range(SLOTS)],
            ids_host=[torch.empty((n, C, K), dtype=torch.int32).pin_memory() for _ in range(SLOTS)],
            boxes_host=[torch.empty((n, C, K, 4), dtype=torch.float32).pin_memory() for _ in range(SLOTS)])
        self._track_n = [None] * SLOTS

    def reset_tracks(self, stream: Optional[int] = None) -> None:
        """Starts every stream (`stream` None), or stream `stream` alone, anew: no tracks, frame count 0, ids from 1, any
        first position.  Ordered after the batches already submitted; the other streams are unaffected."""
        if self._track is None:
            raise RuntimeError("reset_tracks() needs enable_tracking()")
        self._track["tracker"].reset(stream, self._side if self.world > 1 else self._det_stream)

    def tracks(self, ticket: int):
        """(ids int32 [F, C, K], boxes float32 [F, C, K, 4]) of the F frames of the ``submit_images`` batch behind `ticket`, in
        the order of its `frames`: each record's track id (-1: no track, or one not reported in this frame) and, where it
        has an id, its track's state box (ymin, xmin, ymax, xmax) after the frame; pinned host views, valid after
        ``collect(ticket)`` until the ticket's slot is reused.  Frame q is global image q: with several ranks, rank q //
        images_per_batch's image q % images_per_batch.  Ids count from 1 in each stream: with several streams a track is
        identified by (stream, id)."""
        if self._track is None or self._track_n[ticket] is None:
            raise RuntimeError("no tracks for this ticket: call enable_tracking() and give submit_images() its frames")
        self._d2h_done[ticket].synchronize()
        m = self._track_n[ticket]
        return self._track["ids_host"][ticket][:m], self._track["boxes_host"][ticket][:m]

    def _track_slot(self, s: int, st: torch.cuda.Stream, frames: list, streams: Optional[list], last: dict) -> None:
        """Enqueues the tracking of gather slot s's frames (of `streams`; None: all stream 0) on `st`, behind its gathered
        block: rows, positions and streams H2D, one launch of the tracker's kernel (k2y_track_update_streams,
        k2y_bytetrack_update_streams or k2y_ocsort_update_streams), ids and boxes D2H.  `last`: each stream's last position
        in the batch."""
        tk, m, B = self._track, len(frames), self._ipb
        self._track_n[s] = m
        if m == 0:
            return
        self._d2h_done[s].synchronize()       # the slot's last copies out of its pinned inputs have finished
        tk["rows_host"][s].numpy()[:m] = [(q // B) * self.batch + q % B for q in range(m)]
        tk["pos_host"][s].numpy()[:m] = frames
        tk["rows"][:m].copy_(tk["rows_host"][s][:m], non_blocking=True)
        tk["pos"][:m].copy_(tk["pos_host"][s][:m], non_blocking=True)
        if streams is not None:
            tk["streams_host"][s].numpy()[:m] = streams
            tk["streams"][:m].copy_(tk["streams_host"][s][:m], non_blocking=True)
        dets, counts = self.gather.views(s)
        tk["tracker"].update(dets, counts, tk["rows"], tk["pos"], m, tk["ids"], tk["boxes"], st, last,
                             None if streams is None else tk["streams"])
        tk["ids_host"][s][:m].copy_(tk["ids"][:m], non_blocking=True)
        tk["boxes_host"][s][:m].copy_(tk["boxes"][:m], non_blocking=True)

    def enable_png_decode(self) -> None:
        """From now on ``submit_images`` decodes the PNG files the GPU takes (``preprocess.png_gpu_decodable``: non-interlaced,
        not 16-bit grey, sound chunks) on the GPU, with the pixels PIL gives, instead of on the host; ``collect`` raises
        ``K2YError`` naming a PNG whose zlib stream or row filters PIL refuses.  Other PNGs keep the host route."""
        self._gpu_png = True

    def enable_progressive_jpeg_decode(self) -> None:
        """From now on ``submit_images`` decodes the progressive JPEG files the GPU takes
        (``preprocess.progressive_gpu_decodable``) on the GPU, with the pixels PIL gives, instead of on the host; ``collect``
        raises ``K2YError`` naming one whose entropy-coded data was corrupt.  Other progressive files keep the host route."""
        self._gpu_progressive = True

    def set_image_shapes(self, image_hw) -> None:
        """Original (pre-letterbox) image sizes, [batch, 2] (h, w); defaults to the network input size."""
        arr = np.broadcast_to(np.asarray(image_hw, np.float32).reshape(-1, 2), (self.batch, 2))
        self._img_hw.copy_(torch.from_numpy(np.array(arr, dtype=np.float32, order="C", copy=True)))

    # -- device-resident step ---------------------------------------------------------------------------------------
    def _step(self, n: int, image_hw: Optional[torch.Tensor] = None, view_yx: Optional[torch.Tensor] = None, table=None) -> int:
        """Network on the current stream into head set s, decode/NMS on the decode stream into gather slot s, then
        (world > 1) the all-gather on the side stream.  `image_hw`: device [n, 2] original sizes (default: the shared
        ``set_image_shapes`` tensor).  With `view_yx` (device [n, 2] origins) the n inputs are the views of n // V images: the
        decode writes the per-view block and the merge writes the gather slot.  `table` = (device address of the view offsets,
        of the view sides, of the mirror flags or None, images) switches to ``k2y_merge_views_mirror`` with the tiling's options.
        Returns s."""
        s = self._steps % SLOTS
        self._steps += 1
        compute = torch.cuda.current_stream(self.device_index)
        if self._head_sets is None:
            self._head_sets = [list(self.engine.head_buffers), self.engine.new_head_set()]
        # head set s was last read by the decode of two steps ago; that decode wrote gather slot s, too
        compute.wait_event(self._det_done[s])
        self.engine.bind_heads(self._head_sets[s])
        heads = self.engine.run(n)
        self._heads_ready[s].record(compute)
        det = self._det_stream
        det.wait_event(self._heads_ready[s])
        det.wait_event(self._slot_free[s])          # whoever still reads this gather slot (all-gather / D2H two steps ago)
        dets, counts = self.gather.local(s)
        if view_yx is None:
            self.detector.run(heads, self._img_hw[:n] if image_hw is None else image_hw, dets_out=dets, counts_out=counts, stream=det)
        elif table is not None:
            self.detector.run(heads, image_hw, dets_out=self._view_dets, counts_out=self._view_counts, stream=det)
            m = self._merge
            off, sides, mirror, n_images = table
            bordered = m["border"] is not None
            check(lib.k2y_merge_views_mirror(self._view_dets.data_ptr(), self._view_counts.data_ptr(), view_yx.data_ptr(), off,
                                             sides if bordered else None, mirror,
                                             image_hw.data_ptr() if bordered or mirror is not None else None,
                                             m["border"] if bordered else -1.0, m["match"], m["merge"], n_images, self.batch,
                                             self._views, self._nbox, self.gather.C, self.gather.K, m["thresh"], dets.data_ptr(),
                                             counts.data_ptr(), dets.stride(0), counts.stride(0), ctypes.c_void_p(det.cuda_stream)))
        else:
            self.detector.run(heads, image_hw, dets_out=self._view_dets, counts_out=self._view_counts, stream=det)
            check(lib.k2y_merge_views(self._view_dets.data_ptr(), self._view_counts.data_ptr(), view_yx.data_ptr(), n // self._views,
                                      self.batch, self._views, self._nbox, self.gather.C, self.gather.K, self.detector.cfg.iou_thresh,
                                      dets.data_ptr(), counts.data_ptr(), dets.stride(0), counts.stride(0),
                                      ctypes.c_void_p(det.cuda_stream)))
        self._det_done[s].record(det)
        if self.world > 1:
            self._side.wait_event(self._det_done[s])
            self.gather.gather(s, stream=self._side)
            self._gather_done[s].record(self._side)
            self._slot_free[s].record(self._side)
        return s

    def step_device(self, n: Optional[int] = None, pipelined: bool = False):
        """Network + decode/NMS (+ all-gather) on the bound device input; asynchronous.  Returns the gathered
        (dets [world*batch, C, K, 6] int32, counts [world*batch, C]) device views.  ``pipelined=False``: the current stream
        waits for them (use them like any other result of the stream).  ``pipelined=True``: the current stream does NOT wait,
        so the next step's convolutions overlap this step's decode; the views are complete once the stream has passed
        ``wait_gathered()`` (or after a device synchronise), and stay valid for one more ``step_device``."""
        s = self._step(self.batch if n is None else n)
        self._last_slot = s
        if not pipelined:
            self.wait_gathered()
        return self.gather.views(s)

    def wait_gathered(self) -> None:
        """Makes the current stream wait for the decode (and all-gather) of the latest ``step_device``."""
        ev = self._gather_done[self._last_slot] if self.world > 1 else self._det_done[self._last_slot]
        torch.cuda.current_stream(self.device_index).wait_event(ev)

    # -- host API ---------------------------------------------------------------------------------------------------
    def _input_slots(self, u8: bool) -> List[torch.Tensor]:
        if u8:
            if self._in_u8 is None:
                self._in_u8 = [torch.empty(self.engine.input_buffer.shape, dtype=torch.uint8, device=self.engine.input_buffer.device)
                               for _ in range(SLOTS)]
            return self._in_u8
        if self._in_f32 is None:
            self._in_f32 = [torch.empty_like(self.engine.input_buffer) for _ in range(SLOTS)]
        return self._in_f32

    def detect_host(self, x_host: torch.Tensor):
        """x_host: CPU float32 (normalised) or uint8 (raw letterboxed RGB) [batch,H,W,3] tensor, pinned for an
        asynchronous copy.  Returns host tensors (dets, counts) for all images of the job, after a stream synchronise."""
        tk = self.submit(x_host)
        return self.collect(tk)

    def submit(self, x_host: torch.Tensor) -> int:
        """Streaming form of ``detect_host``: enqueue one batch (pinned host float32 or uint8 [n,H,W,3]) and return a
        ticket.  The H2D copy runs on a side stream straight into one of two device input buffers (the network is
        re-pointed at it), so it overlaps the previous batch's kernels; at most two batches are in flight —
        ``collect`` the ticket of batch i-1 before submitting batch i+1."""
        n = x_host.shape[0]
        slot = self._submitted % SLOTS
        self._submitted += 1
        # raw letterboxed RGB (uint8): 4x fewer PCIe bytes, the normalisation (img / max(img)) is fused into the first conv
        buf = self._input_slots(x_host.dtype == torch.uint8)[slot]
        self._copy_stream.wait_event(self._in_free[slot])
        with torch.cuda.stream(self._copy_stream):
            buf[:n].copy_(x_host, non_blocking=True)
            self._h2d_done[slot].record(self._copy_stream)
        self._jpeg_idx[self._steps % SLOTS] = []
        self._png_idx[self._steps % SLOTS] = []
        self._prog_idx[self._steps % SLOTS] = []
        t = self._run_slot(slot, buf, n, None, None)
        self._rendered_slot[t] = False
        self._track_n[t] = None
        return t

    def enable_rendering(self, quality: int = 75, font_path: str = "asset/FiraMono-Medium.otf", colormap=None, *,
                         tracks: bool = False) -> None:
        """From now on every ``submit_images`` batch also has its local records drawn onto its original images (as
        ``draw.draw_detections`` draws them, ``render.render_detections_device``) and encoded as JPEG files (as PIL saves them at
        `quality`, ``render.JpegEncoder``), on the decode stream behind the NMS; ``rendered(ticket)`` returns them after
        ``collect``.  `colormap`: RGB triples per class (default ``Helper.colormap``, 80 classes).  Records and ``collect``
        are unchanged.  ``submit_images`` then refuses an image with more than ``render.JPEG_MAX_DIMENSION`` (65500) rows or
        columns, which no JPEG file can hold.

        With `tracks` each image is drawn with its tracks instead, as ``draw.draw_tracks`` draws the frame's rows of
        ``tracks(ticket)`` (``render.render_tracks_device``): every record with a track id, its track box in colour
        ``colormap[id % len(colormap)]``, labelled ``"{class:2d} #{id}"``.  An image that is not one of the batch's frames is
        encoded undrawn.  ``submit_images`` then needs tracking on (``enable_tracking``)."""
        from .helper import _COLORMAP
        from .render import MAX_CLASSES, JpegEncoder, LabelAtlas, TrackLabelAtlas, color_table, track_color_table
        colormap = _COLORMAP if colormap is None else colormap
        C = self.gather.C
        if C > len(colormap) and not tracks:
            raise ValueError(f"class_num {C} exceeds the colormap's {len(colormap)} classes")
        if not 1 <= int(quality) <= 100:
            raise ValueError(f"quality {quality} is outside 1..100")
        dev = torch.device("cuda", self.device_index)
        if tracks:
            if C > MAX_CLASSES:
                raise ValueError(f"class_num {C}: tracks are drawn for at most {MAX_CLASSES} classes")
            atlas, colors = TrackLabelAtlas(font_path), track_color_table(colormap, dev)
        else:
            atlas, colors = LabelAtlas(C, font_path), color_table(colormap, C, dev)
        self._render = dict(quality=int(quality), atlas=atlas, colors=colors, tracks=bool(tracks),
                            encoders=[JpegEncoder(dev) for _ in range(SLOTS)])

    def rendered(self, ticket: int) -> List[bytes]:
        """The JPEG files of this rank's images of the ``submit_images`` batch behind `ticket`, with its records drawn on them;
        valid after ``collect(ticket)`` until the ticket's slot is reused."""
        if self._render is None or not self._rendered_slot[ticket]:
            raise RuntimeError("no rendered files for this ticket: call enable_rendering() before submit_images()")
        self._render_done[ticket].synchronize()
        return self._render["encoders"][ticket].fetch()

    def _render_slot(self, slot: int, s: int, layout: BatchLayout) -> None:
        """Draws gather slot s's local records onto input slot `slot`'s originals and encodes them, on the decode stream."""
        from .render import render_packed
        r = self._render
        det = self._det_stream
        det.wait_event(self._h2d_done[slot])     # the originals are in place (already implied by the network's wait)
        staging = self._staging[slot]
        dets, counts = self.gather.local(s)
        n = len(layout)
        with torch.cuda.stream(det):
            render_packed(staging.dev.data_ptr(), layout.offsets, layout.hw, dets[:n], counts[:n], r["atlas"], r["colors"],
                          staging.dev.device, det)
            r["encoders"][s].enqueue(staging.dev.data_ptr(), layout.offsets, layout.hw, r["quality"], det)
        self._render_done[s].record(det)
        self._render_free[slot].record(det)

    def _render_tracks_slot(self, slot: int, s: int, layout: BatchLayout, st: torch.cuda.Stream) -> None:
        """Draws the tracks of this rank's frames of gather slot s onto input slot `slot`'s originals and encodes them, on
        `st`, the stream that ran the slot's tracking, right behind it.  The device ids and boxes hold one batch's tracks:
        the next batch's tracking, enqueued on `st` by a later ``submit_images``, overwrites them only after this render."""
        from .render import render_tracks_packed
        r, tk = self._render, self._track
        st.wait_event(self._h2d_done[slot])      # the originals are in place (already implied by the network's wait)
        staging = self._staging[slot]
        n = len(layout)
        q0, row0 = self.rank * self._ipb, self.rank * self.batch    # this rank's first frame and its gathered row
        drawn = min(n, max(0, (self._track_n[s] or 0) - q0))        # images past the batch's frames are encoded undrawn
        with torch.cuda.device(staging.dev.device):
            if drawn:
                _, counts = self.gather.views(s)
                render_tracks_packed(staging.dev.data_ptr(), layout.offsets[:drawn], layout.hw[:drawn], counts[row0:row0 + drawn],
                                     tk["ids"][q0:q0 + drawn], tk["boxes"][q0:q0 + drawn], r["atlas"], r["colors"],
                                     staging.dev.device, st)
            r["encoders"][s].enqueue(staging.dev.data_ptr(), layout.offsets, layout.hw, r["quality"], st)
        self._render_done[s].record(st)
        self._render_free[slot].record(st)

    def submit_images(self, images: Sequence[np.ndarray], frames: Optional[Sequence[int]] = None,
                      streams: Optional[Sequence[int]] = None) -> int:
        """Streaming form for raw images: `images` is a list of n <= ``images_per_batch`` host numpy uint8 [h, w, 3] RGB arrays of any sizes, or
        image files (``bytes``, ``bytearray``, ``memoryview``): baseline JPEGs are decoded on the GPU on the copy stream in front
        of the letterbox, other files on the host inside this call (``preprocess.BatchLayout``).
        They are packed into the input slot's pinned staging buffer, copied to the GPU in one H2D copy and letterboxed in one
        launch into the slot's uint8 input buffer (``k2y_letterbox_u8_batch``, which also writes the slot's device
        ``image_hw`` the decode reads), on the copy stream, overlapping the previous batch's network.  The network runs the n
        images.  Returns a ticket for ``collect``, which returns the n images' records (world > 1: the gathered blocks of every
        rank, rank r's images from row r * batch), or raises ``K2YError`` naming the JPEGs whose entropy-coded data was corrupt
        (their records would come from undefined pixels).  Same flow control as ``submit``.  Bad input raises ``ValueError``
        before anything is enqueued.

        With ``enable_tracking`` `frames` is required: the stream positions of the global batch's frames in gathered-row order
        (global image q is rank q // images_per_batch's image q % images_per_batch; images past len(frames) are not frames),
        increasing along the stream.  Every rank gives the same list.  With ``enable_tracking(streams=S)``, S > 1, `streams`
        is required too: each frame's stream in 0..S-1, in the same order as `frames` (left out, every frame is stream 0);
        positions increase along each stream, and the streams are independent of one another."""
        viewed = self._tiling is not None or self._flip
        if viewed and isinstance(images, (list, tuple)) and len(images) > self.images_per_batch:
            raise ValueError(f"{len(images)} images of {self._views} views do not fit a batch of {self.batch}")
        layout = BatchLayout(images, self.in_hw, self._tiling, gpu_png=self._gpu_png, gpu_progressive=self._gpu_progressive,
                             merge_table=self._merge is not None, flip=self._flip)
        n = len(layout)
        if n > self.batch:
            raise ValueError(f"{n} images do not fit a batch of {self.batch}")
        if (frames is None) != (self._track is None):
            raise ValueError("submit_images takes frames= exactly when tracking is on (enable_tracking)")
        last = None
        if frames is not None:
            tracker = self._track["tracker"]
            if streams is None and tracker.streams > 1:
                raise ValueError(f"submit_images takes streams= when tracking {tracker.streams} streams")
            frames, stream_list, last = check_positions(frames, streams, tracker.last_positions)
            streams = None if streams is None else stream_list
            if len(frames) > self.world * self._ipb or (self.world == 1 and len(frames) > n):
                raise ValueError(f"{len(frames)} frame positions for {n} images per rank of {self.world} ranks")
        elif streams is not None:
            raise ValueError("submit_images takes streams= only with frames= (enable_tracking)")
        if self._render is not None and self._render["tracks"]:
            if self._track is None:
                raise ValueError("enable_rendering(tracks=True) draws the tracks: call enable_tracking() too")
            for h in sorted({h for h, _ in layout.hw.tolist()}):
                self._render["atlas"].host(h)   # builds the glyphs of each new font size here: a refused font raises now
        if self._render is not None:
            from .render import JPEG_MAX_DIMENSION
            for i, (h, w) in enumerate(layout.hw.tolist()):
                if h > JPEG_MAX_DIMENSION or w > JPEG_MAX_DIMENSION:
                    raise ValueError(f"image {i} is {h}x{w}: a rendered JPEG file has at most {JPEG_MAX_DIMENSION} rows and columns")
        slot = self._submitted % SLOTS
        buf = self._input_slots(True)[slot]
        dev = buf.device
        if self._staging is None:
            self._staging = [Staging(dev, self._copy_stream) for _ in range(SLOTS)]
            self._slot_hw = [torch.empty((self.batch, 2), dtype=torch.float32, device=dev) for _ in range(SLOTS)]
        self._h2d_done[slot].synchronize()     # the last copy out of this slot's pinned buffer has finished: repack / grow it
        self._submitted += 1
        self._copy_stream.wait_event(self._in_free[slot])
        self._copy_stream.wait_event(self._hw_free[slot])
        self._copy_stream.wait_event(self._render_free[slot])    # the last render read this slot's originals
        s = self._steps % SLOTS                  # the gather slot this batch's step will use
        with torch.cuda.device(dev):
            letterbox_packed(layout, images, self._staging[slot], buf, self._slot_hw[slot],
                             self._slot_yx[slot] if viewed else None)
            self._jpeg_idx[s] = [i for i, _ in layout.jpeg]
            if layout.jpeg:             # the status words travel to the host before the network starts on this slot
                with torch.cuda.stream(self._copy_stream):
                    self._jpeg_status[s][:len(layout.jpeg)].copy_(self._staging[slot].status[:len(layout.jpeg)], non_blocking=True)
            self._png_idx[s] = [i for i, _ in layout.png]
            if layout.png:
                with torch.cuda.stream(self._copy_stream):
                    self._png_status[s][:len(layout.png)].copy_(self._staging[slot].png_status[:len(layout.png)], non_blocking=True)
            self._prog_idx[s] = [i for i, _ in layout.progressive]
            if layout.progressive:
                np_ = len(layout.progressive)
                with torch.cuda.stream(self._copy_stream):
                    self._prog_status[s][:np_].copy_(self._staging[slot].progressive_status[:np_], non_blocking=True)
        self._h2d_done[slot].record(self._copy_stream)
        nv = layout.n_views
        table = None
        if layout.merge_table_at is not None:     # the view offsets, sides and mirror flags, where the H2D copy put them
            at = self._staging[slot].dev.data_ptr() + layout.merge_table_at
            table = (at, at + 4 * (n + 1), at + 4 * (n + 1 + nv) if self._flip else None, n)
        draw_tracks = self._render is not None and self._render["tracks"]
        t = self._run_slot(slot, buf, nv, self._slot_hw[slot][:nv], n if self.world == 1 else None,
                           self._slot_yx[slot][:nv] if viewed else None, table, frames, streams, last,
                           (lambda s, st: self._render_tracks_slot(slot, s, layout, st)) if draw_tracks else None)
        self._rendered_slot[t] = self._render is not None
        if self._render is not None and not draw_tracks:
            with torch.cuda.device(dev):
                self._render_slot(slot, t, layout)
        return t

    def _run_slot(self, slot: int, buf: torch.Tensor, n: int, image_hw: Optional[torch.Tensor], rows: Optional[int],
                  view_yx: Optional[torch.Tensor] = None, table=None, frames: Optional[list] = None,
                  streams: Optional[list] = None, last: Optional[dict] = None, after_track=None) -> int:
        """Network + decode (+ all-gather) of input slot `slot` once its H2D is done, then (with `frames`) the tracking, then
        the D2H of the records, then ``after_track(gather slot, stream)`` on the same stream (the track drawing)."""
        compute = torch.cuda.current_stream(self.device_index)
        compute.wait_event(self._h2d_done[slot])
        self.engine.bind_input(buf)
        s = self._step(n, image_hw, view_yx, table)
        self._in_free[slot].record(compute)
        self._hw_free[slot].record(self._det_stream)
        self._rows[s] = rows
        # D2H of the gathered blocks: behind the all-gather on the side stream (world > 1), else behind the decode
        st = self._side if self.world > 1 else self._det_stream
        with torch.cuda.stream(st):
            if frames is not None:
                self._track_slot(s, st, frames, streams, last)
            self._host[s].copy_(self.gather.bufs[s], non_blocking=True)
            self._d2h_done[s].record(st)
            if after_track is not None:
                after_track(s, st)
            self._slot_free[s].record(st)
        return s

    def collect(self, ticket: int):
        """Blocks until the batch behind `ticket` is on the host; returns (dets, counts) pinned host views (valid
        until the ticket's slot is reused two submits later).  Raises ``K2YError`` when a JPEG of a ``submit_images`` batch had
        corrupt entropy-coded data."""
        self._d2h_done[ticket].synchronize()      # behind the network, which waited for the batch's decode and status copy
        if self._rendered_slot[ticket]:
            self._render_done[ticket].synchronize()   # the files' lengths are on the host
        if self._jpeg_idx[ticket]:
            idx = self._jpeg_idx[ticket]
            check_jpeg_status(self._jpeg_status[ticket][:len(idx)].numpy(), idx)
        if self._png_idx[ticket]:
            idx = self._png_idx[ticket]
            check_png_status(self._png_status[ticket][:len(idx)].numpy(), idx)
        if self._prog_idx[ticket]:
            idx = self._prog_idx[ticket]
            check_progressive_status(self._prog_status[ticket][:len(idx)].numpy(), idx)
        dets, counts = DetectionGather.split(self._host[ticket], self.gather.C, self.gather.K, DET_WORDS)
        n = self._rows[ticket]
        return (dets, counts) if n is None else (dets[:n], counts[:n])

    def launches_per_step(self) -> int:
        return self.engine.launches_per_run() + 2  # + the decode scan and the per-class NMS kernel

    @staticmethod
    def records(dets: torch.Tensor, counts: torch.Tensor) -> List[list]:
        return KerasDetector.to_host(dets, counts)


class LanedPipeline:
    """Several batches in flight: ``lanes`` DetectionPipelines (own engine + activation arena, own streams, one shared NCCL
    communicator) fed round-robin, each on its own compute stream.  Consecutive batches are independent, so batch i+1's
    bandwidth-bound early layers run beside batch i's small-grid late layers — the multi-stream serving form of the same
    per-batch work; every batch still goes through the same kernels with the same batch size.  With ``sm_split`` (default) every
    lane sizes its persistent tensor-core grids for 1/lanes of the SMs, so the lanes' kernels share the GPU side by side.

    ``bind_input(x)`` / ``step_device()`` / ``wait_all()`` for device-resident inputs, ``submit`` / ``collect`` for pinned
    host batches and ``submit_images`` / ``collect`` for raw host images of any size (tickets carry the lane)."""

    def __init__(self, lanes: int, *args, sm_split: bool = True, sm_limit: Optional[int] = None, max_queued: Optional[int] = None, **kw):
        if lanes < 1:
            raise ValueError("lanes must be >= 1")
        first = DetectionPipeline(*args, **kw)
        self.lanes: List[DetectionPipeline] = [first] + [DetectionPipeline(*args, comm=first.gather.comm, **kw) for _ in range(lanes - 1)]
        self.batch, self.world, self.rank, self.device_index = first.batch, first.world, first.rank, first.device_index
        dev = torch.device("cuda", self.device_index)
        self._streams = [torch.cuda.Stream(device=dev) for _ in self.lanes]
        self._fork = torch.cuda.Event()
        self._next = 0          # next lane for step_device
        self._next_host = 0     # next lane for submit
        self._ran = [False] * lanes
        # host-side flow control of step_device: at most `max_queued` batches issued and not yet through their network — a bounded
        # queue, as a server has.  Default 2 per lane (= the gather / head-set slots of a lane, and what submit/collect allows):
        # the GPU always has a full step queued behind the running one, and the host never runs further ahead.
        self.max_queued = max(lanes, int(max_queued)) if max_queued is not None else 2 * lanes
        self._flow_events = [torch.cuda.Event() for _ in range(self.max_queued)]
        self._flow_pending = 0
        self._issued = 0
        # each lane plans its persistent tensor-core kernels for 1/lanes of the SMs: two lanes' one-CTA-per-SM grids then run
        # side by side
        self.sm_limit = 0
        if sm_limit is not None:
            self.sm_limit = int(sm_limit)
        elif sm_split and lanes > 1:
            self.sm_limit = torch.cuda.get_device_properties(dev).multi_processor_count // lanes
        if self.sm_limit:
            for ln in self.lanes:
                ln.engine.set_sm_limit(self.sm_limit)

    def set_weights(self, weights) -> None:
        for ln in self.lanes:
            ln.engine.set_weights(weights)

    def set_math(self, mode) -> None:
        for ln in self.lanes:
            ln.engine.set_math(mode)

    def set_image_shapes(self, image_hw) -> None:
        for ln in self.lanes:
            ln.set_image_shapes(image_hw)

    def bind_input(self, x: torch.Tensor) -> None:
        """Device input of the NEXT ``step_device`` (float32 or uint8 [batch,H,W,3])."""
        self.lanes[self._next % len(self.lanes)].engine.bind_input(x)

    def step_device(self, n: Optional[int] = None):
        """One batch on the next lane (asynchronous, on the lane's stream, ordered after the caller's current stream).  The
        returned views are complete after ``wait_all()`` and stay valid until that lane has run two more batches."""
        k = self._next % len(self.lanes)
        self._next += 1
        cur = torch.cuda.current_stream(self.device_index)
        self._fork.record(cur)
        st = self._streams[k]
        st.wait_event(self._fork)
        slot = self._issued % self.max_queued
        if self._issued >= self.max_queued:
            self._flow_events[slot].synchronize()     # the batch issued max_queued steps ago has left its network
        with torch.cuda.stream(st):
            views = self.lanes[k].step_device(n, pipelined=True)
            self._flow_events[slot].record(st)
        self._issued += 1
        self._ran[k] = True
        return views

    def wait_all(self) -> None:
        """Makes the current stream wait for everything issued with ``step_device`` so far (decode / all-gather of every lane)."""
        for k, ln in enumerate(self.lanes):
            if self._ran[k]:
                ln.wait_gathered()

    def submit(self, x_host: torch.Tensor):
        k = self._next_host % len(self.lanes)
        self._next_host += 1
        with torch.cuda.stream(self._streams[k]):
            return (k, self.lanes[k].submit(x_host))

    def submit_images(self, images: Sequence[np.ndarray]):
        """``DetectionPipeline.submit_images`` on the next lane (round-robin, shared with ``submit``)."""
        k = self._next_host % len(self.lanes)
        with torch.cuda.stream(self._streams[k]):
            t = self.lanes[k].submit_images(images)
        self._next_host += 1
        return (k, t)

    def collect(self, ticket):
        k, t = ticket
        return self.lanes[k].collect(t)

    def enable_rendering(self, quality: int = 75, font_path: str = "asset/FiraMono-Medium.otf", colormap=None, *,
                         tracks: bool = False) -> None:
        """``DetectionPipeline.enable_rendering`` on every lane.  Not with `tracks`: the lanes do not track."""
        if tracks:
            raise NotImplementedError("track drawing needs tracking, which runs on a DetectionPipeline; a LanedPipeline's lanes "
                                      "cannot order one stream's frames")
        for ln in self.lanes:
            ln.enable_rendering(quality, font_path, colormap)

    def enable_png_decode(self) -> None:
        """``DetectionPipeline.enable_png_decode`` on every lane."""
        for ln in self.lanes:
            ln.enable_png_decode()

    def enable_progressive_jpeg_decode(self) -> None:
        """``DetectionPipeline.enable_progressive_jpeg_decode`` on every lane."""
        for ln in self.lanes:
            ln.enable_progressive_jpeg_decode()

    def enable_tiling(self, rows: Optional[int] = None, cols: Optional[int] = None, overlap: float = 0.2, *, tile_size=None,
                      images_per_batch: Optional[int] = None, match: str = "iou", merge: str = "suppress",
                      match_thresh: Optional[float] = None, border: Optional[float] = None) -> None:
        """``DetectionPipeline.enable_tiling`` on every lane."""
        for ln in self.lanes:
            ln.enable_tiling(rows, cols, overlap, tile_size=tile_size, images_per_batch=images_per_batch, match=match, merge=merge,
                             match_thresh=match_thresh, border=border)

    def enable_tracking(self, max_age: int = 1, min_hits: int = 3, iou_thresh: float = 0.3, **kw) -> None:
        """Not available: the lanes would have to hand one stream's frames over in order."""
        raise NotImplementedError("tracking runs on a DetectionPipeline; a LanedPipeline's lanes cannot order one stream's frames")

    def enable_flip(self, *, match: Optional[str] = None, merge: Optional[str] = None, match_thresh: Optional[float] = None,
                    border: Optional[float] = None) -> None:
        """``DetectionPipeline.enable_flip`` on every lane."""
        for ln in self.lanes:
            ln.enable_flip(match=match, merge=merge, match_thresh=match_thresh, border=border)

    @property
    def images_per_batch(self) -> int:
        return self.lanes[0].images_per_batch

    def rendered(self, ticket) -> List[bytes]:
        k, t = ticket
        return self.lanes[k].rendered(t)

    def in_flight_limit(self) -> int:
        """Batches that may be submitted before the oldest must be collected."""
        return SLOTS * len(self.lanes)

    def launches_per_step(self) -> int:
        return self.lanes[0].launches_per_step()
