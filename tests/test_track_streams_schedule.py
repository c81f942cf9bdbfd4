"""The multi-stream schedule and checks on the host: ``serve.interleave`` puts every frame of every sequence in once, in
order along each slot's stream, never shares a slot within a batch and resets a slot before it is reused; serve.py refuses
mixed, repeated and same-stem inputs; ``track.check_positions`` checks positions per stream."""
import pytest

import serve
from k210_yolo_framework_b200.track import check_positions


def _check(lengths, slots, G):
    sched = serve.interleave(lengths, slots, G)
    seen = [[] for _ in lengths]
    holder = {}                     # slot -> the sequence it holds
    last_pos = {}                   # slot -> the last (sequence, frame) of its stream
    for g, (frames, resets) in enumerate(sched):
        assert 0 < len(frames) <= G
        for slot in resets:         # a slot is reset only when it held another sequence, which has ended
            assert slot in holder
            i = holder.pop(slot)
            assert len(seen[i]) == lengths[i]
            last_pos.pop(slot)
        in_batch = {}
        for i, k, slot in frames:
            assert 0 <= slot < slots
            assert in_batch.setdefault(slot, i) == i            # one sequence per slot within a batch
            assert holder.setdefault(slot, i) == i              # a slot changes sequence only through a reset
            assert last_pos.get(slot, (i, -1)) < (i, k)         # positions increase along the slot's stream
            last_pos[slot] = (i, k)
            seen[i].append(k)
        if g < len(sched) - 1 and len(frames) < G:     # a short batch: every sequence active in it has ended in it
            assert all(len(seen[i]) == lengths[i] for i in in_batch.values())
    assert seen == [list(range(n)) for n in lengths]   # every frame once, in frame order
    return sched


@pytest.mark.parametrize("lengths,slots,G", [
    ([7], 1, 4), ([9, 3, 0, 14, 1, 6], 1, 4), ([9, 3, 0, 14, 1, 6], 3, 4), ([9, 3, 0, 14, 1, 6], 2, 5),
    ([9, 3, 0, 14, 1, 6], 6, 4), ([9, 3, 14, 1, 6], 8, 3), ([5, 5, 5], 3, 1), ([40, 2, 2, 2, 2, 2, 2], 2, 7), ([], 3, 4),
    ([0, 0], 2, 4), ([100, 50, 75, 1], 4, 32)])
def test_interleave_schedules_every_frame_once_per_stream_order(lengths, slots, G):
    sched = _check(lengths, slots, G)
    if slots >= len(lengths):       # every sequence active at once: batches are full but the last
        assert all(len(f) == G for f, _ in sched[:-1])
        assert not any(r for _, r in sched)


def test_interleave_with_one_slot_is_the_sequential_run():
    """One slot: each sequence in batches of G with a short last batch, the next sequence after a reset of slot 0."""
    sched = serve.interleave([5, 3], 1, 2)
    assert sched == [([(0, 0, 0), (0, 1, 0)], []), ([(0, 2, 0), (0, 3, 0)], []), ([(0, 4, 0)], []),
                     ([(1, 0, 0), (1, 1, 0)], [0]), ([(1, 2, 0)], [])]


def test_interleave_round_robin_and_slot_reuse():
    sched = serve.interleave([2, 4, 3], 2, 3)
    assert sched[0] == ([(0, 0, 0), (1, 0, 1), (0, 1, 0)], [])
    # sequence 0 ended in batch 0: slot 0 is reset and taken by sequence 2 from batch 1 only
    assert sched[1] == ([(1, 1, 1), (2, 0, 0), (1, 2, 1)], [0])
    assert sched[2] == ([(2, 1, 0), (1, 3, 1), (2, 2, 0)], [])
    assert len(sched) == 3


def test_interleave_refuses_bad_sizes():
    for slots, G in ((0, 4), (2, 0)):
        with pytest.raises(ValueError):
            serve.interleave([3], slots, G)


def test_check_positions_per_stream():
    pos, strm, last = check_positions([500, 0, 501, 1, 0], [0, 1, 0, 1, 2], [499, None, None])
    assert (pos, strm, last) == ([500, 0, 501, 1, 0], [0, 1, 0, 1, 2], {0: 501, 1: 1, 2: 0})
    assert check_positions([3, 4], None, [2]) == ([3, 4], [0, 0], {0: 4})
    # the same positions spread over different streams are accepted
    assert check_positions([7, 7, 7], [0, 1, 2], [None, 6, None])[2] == {0: 7, 1: 7, 2: 7}
    for positions, streams, last in (
            ([5, 5], [0, 0], [None]),                # not increasing within its stream
            ([4, 3], [1, 1], [None, None]),
            ([10], [0], [10]),                       # not after the stream's last position
            ([0], [2], [None, None]),                # stream out of range
            ([0], [-1], [None, None]),
            ([-1], None, [None]),                    # negative position
            ([1, 2], [0], [None])):                  # a stream per position
        with pytest.raises(ValueError):
            check_positions(positions, streams, last)


def _video(path):
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_bytes(b"RIFF" + bytes(4) + b"AVI " + bytes(32))     # recognised by content; never opened here
    return str(path)


def _parse(argv):
    return serve.build_parser().parse_args(["model.h5"] + argv)


def test_parser_takes_several_videos_and_refuses_bad_input(tmp_path):
    a, b = _video(tmp_path / "a.avi"), _video(tmp_path / "b.avi")
    same_stem = _video(tmp_path / "other" / "a.avi")
    images = tmp_path / "imgs"
    images.mkdir()
    assert _parse([a]).images == [a]
    assert _parse([a, b, "--track", "--draw", str(tmp_path / "out")]).images == [a, b]
    assert _parse([a, same_stem]).images == [a, same_stem]         # one stem is fine without --draw
    for argv in ([a, str(images)], [str(images), a], [a, b, a], [a, str(tmp_path / "a.avi")],
                 [a, same_stem, "--draw", str(tmp_path / "out")], [str(images), "--track"]):
        with pytest.raises(SystemExit):
            _parse(argv)


def test_draw_paths_refuses_duplicate_stems(tmp_path):
    assert serve.draw_paths(["x/a.avi", "y/b.mp4"], "out", ".avi") == ["out/a.avi", "out/b.avi"]
    with pytest.raises(ValueError, match="a.avi"):
        serve.draw_paths(["x/a.avi", "y/a.mp4"], "out", ".avi")
    assert serve.draw_paths(["x/a.png"], "o") == ["o/a.jpg"]
