"""oracle/mot_ref.py, the MOTChallenge protocol: the restatement against its literal numpy / scipy form, the by-rounds CLEAR
against the sequential loop, the isolated-positives shortcut against a full assignment, the component-wise IDTP against
scipy on the square matrix, hand-worked cases, and the sequence loader."""
import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from mot_sequences import blocks, sequence
from oracle import mot_ref


def _trk(frames):
    ids, boxes, dets, counts = blocks(frames)
    return mot_ref.tracker_rows(range(len(frames)), ids, boxes, dets, counts, 14)


@pytest.mark.parametrize("seed,benchmark", [(0, "MOT17"), (1, "MOT20"), (2, "MOT15"), (3, "MOT16"), (4, "MOT17")])
def test_restatement_equals_the_literal_form(seed, benchmark):
    rng = np.random.default_rng(seed)
    gt, frames = sequence(rng, 80, ambiguous=0.4, benchmark=benchmark)
    trk = _trk(frames)
    a = mot_ref.evaluate("s", gt, trk, 80, benchmark)
    b = mot_ref.evaluate_literal(gt, trk, 80, benchmark)
    assert a == b
    assert a["IDSW"] > 0 and a["Frag"] > 0 and a["TP"] > 500


def _chain(L):
    """Two pedestrians on one box and two tracks on one box, the tracks' rows swapped every frame and a third track beside:
    every frame's assignment is a tie that only the previous frame's matches break."""
    gt, trk = [], []
    for f in range(1, L + 1):
        gt += [[f, 1, 100, 100, 50, 100, 1, 1], [f, 2, 100, 100, 50, 100, 1, 1]]
        pair = [[f, 10, 101, 100, 50, 100, 1], [f, 11, 101, 100, 50, 100, 1]]
        trk += (pair if f % 2 else pair[::-1]) + ([[f, 12, 100, 101, 50, 100, 1]] if f % 3 == 0 else [])
    return np.array(gt, np.float64), np.array(trk, np.float64)


@pytest.mark.parametrize("seed", range(4))
def test_rounds_equal_the_sequential_loop(seed):
    gt, frames = sequence(np.random.default_rng(10 + seed), 120, ambiguous=0.5)
    trk = _trk(frames)
    fr = mot_ref.preprocess(gt, trk, 120)
    pairs, rounds = mot_ref.clear_pairs_by_rounds(fr)
    assert pairs == mot_ref.clear_pairs(fr)
    assert rounds >= 2


def test_rounds_on_a_chain_where_every_frame_depends_on_the_one_before():
    gt, trk = _chain(40)
    fr = mot_ref.preprocess(gt, trk, 40)
    pairs, rounds = mot_ref.clear_pairs_by_rounds(fr)
    assert pairs == mot_ref.clear_pairs(fr)
    assert rounds > 20
    a = mot_ref.evaluate("c", gt, trk, 40, by_rounds=True)
    assert a.pop("rounds") == rounds
    assert a == mot_ref.evaluate_literal(gt, trk, 40)
    assert a["IDSW"] == 0


def test_isolated_positives_need_no_assignment():
    rng = np.random.default_rng(5)
    n = 0
    for seed in range(3):
        gt, frames = sequence(np.random.default_rng(seed), 60, ambiguous=0.3)
        for fr in mot_ref.preprocess(gt, _trk(frames), 60):
            if not fr.gids or not fr.tids:
                continue
            prev = {g: t for g in fr.gids for t in fr.tids if rng.random() < 0.2}
            score = mot_ref.clear_score(fr, prev)
            if mot_ref.isolated(score):
                n += 1
                assert mot_ref.assign(score) == mot_ref.assign(score, shortcut=False)
    assert n > 50


def test_component_idtp_equals_scipy_on_the_square_matrix():
    rng = np.random.default_rng(3)
    for _ in range(30):
        G, T = int(rng.integers(1, 12)), int(rng.integers(1, 15))
        pot = rng.integers(0, 4, (G, T)) * (rng.random((G, T)) < 0.3)
        frames = []
        for g in range(G):
            for t in range(T):
                for _ in range(int(pot[g, t])):
                    frames.append(mot_ref.Frame([g], [t], [[1.0]]))
        gcount = pot.sum(1) + rng.integers(0, 3, G)
        tcount = pot.sum(0) + rng.integers(0, 3, T)
        fp, fn = np.zeros((G + T, G + T)), np.zeros((G + T, G + T))
        fp[G:, :T] = 1e10
        fn[:G, T:] = 1e10
        for g in range(G):
            fn[g, :T] = gcount[g]
            fn[g, T + g] = gcount[g]
        for t in range(T):
            fp[:G, t] = tcount[t]
            fp[t + G, t] = tcount[t]
        fn[:G, :T] -= pot
        fp[:G, :T] -= pot
        r, c = linear_sum_assignment(fn + fp)
        assert mot_ref.identity(frames) == int(gcount.sum()) - int(fn[r, c].sum())


# -- hand-worked cases ---------------------------------------------------------------------------------------------------------
A = [100.0, 100.0, 50.0, 100.0]


def _shift(box, dx):
    return [box[0] + dx, box[1], box[2], box[3]]


def _ev(gt, trk, L, benchmark="MOT17"):
    gt, trk = np.array(gt, np.float64).reshape(-1, 8), np.array(trk, np.float64).reshape(-1, 7)
    d = mot_ref.evaluate("hand", gt, trk, L, benchmark)
    r = mot_ref.evaluate("hand", gt, trk, L, benchmark, by_rounds=True)
    r.pop("rounds")
    assert d == r == mot_ref.evaluate_literal(gt, trk, L, benchmark)
    return d


def test_perfect_tracking():
    B = _shift(A, 300)
    gt = [[f, g, *box, 1, 1] for f in (1, 2, 3) for g, box in ((1, A), (2, B))]
    trk = [[f, 10 + g, *box, 1] for f in (1, 2, 3) for g, box in ((1, A), (2, B))]
    d = _ev(gt, trk, 3)
    assert d["MOTA"] == d["IDF1"] == d["MOTP"] == 1.0
    assert (d["TP"], d["FP"], d["FN"], d["IDSW"], d["Frag"], d["MT"], d["IDTP"]) == (6, 0, 0, 0, 0, 2, 6)


def test_one_id_switch():
    gt = [[f, 1, *A, 1, 1] for f in range(1, 5)]
    trk = [[f, 10 if f < 3 else 11, *A, 1] for f in range(1, 5)]
    d = _ev(gt, trk, 4)
    assert (d["TP"], d["IDSW"], d["Frag"], d["IDTP"], d["IDFP"], d["IDFN"]) == (4, 1, 0, 2, 2, 2)
    assert d["MOTA"] == 0.75 and d["IDF1"] == 0.5


def test_a_fragment():
    gt = [[f, 1, *A, 1, 1] for f in range(1, 6)]
    trk = [[f, 10, *(A if f != 3 else _shift(A, 500)), 1] for f in range(1, 6)]
    d = _ev(gt, trk, 5)
    assert (d["TP"], d["FP"], d["FN"], d["IDSW"], d["Frag"], d["MT"], d["PT"], d["ML"]) == (4, 1, 1, 0, 1, 0, 1, 0)
    assert d["MOTA"] == 0.6


def test_the_continuity_bonus_keeps_a_match_over_a_higher_iou_rival():
    gt = [[1, 1, *A, 1, 1], [2, 1, *A, 1, 1]]
    trk = [[1, 10, *A, 1], [2, 10, *_shift(A, 12), 1], [2, 11, *_shift(A, 2), 1]]
    d = _ev(gt, trk, 2)
    assert (d["TP"], d["FP"], d["IDSW"]) == (2, 1, 0)
    assert d["MOTP_sum"] == 1.0 + mot_ref.iou(A, _shift(A, 12))


def test_frames_without_gt_or_tracker_rows_keep_continuity():
    gt = [[1, 1, *A, 1, 1], [2, 1, *A, 1, 1], [4, 1, *A, 1, 1]]
    trk = [[1, 10, *A, 1], [3, 10, *A, 1], [4, 10, *_shift(A, 12), 1], [4, 11, *_shift(A, 2), 1]]
    d = _ev(gt, trk, 4)
    assert (d["TP"], d["FP"], d["FN"], d["IDSW"], d["Frag"]) == (2, 2, 1, 0, 0)


def test_a_tracker_box_on_a_distractor_is_removed_and_one_on_a_zero_marked_pedestrian_is_a_false_positive():
    B, C = _shift(A, 300), _shift(A, 600)
    gt = [[1, 1, *A, 1, 1], [1, 2, *B, 1, 7], [1, 3, *C, 0, 1]]
    trk = [[1, 10, *A, 1], [1, 11, *B, 1], [1, 12, *C, 1]]
    d = _ev(gt, trk, 1)
    assert (d["TP"], d["FP"], d["FN"], d["tracker_rows"], d["gt_rows"]) == (1, 1, 0, 2, 1)


def test_mot15_has_no_distractor_removal():
    B = _shift(A, 300)
    gt = [[1, 1, *A, 1, 1], [1, 2, *B, 1, 7]]
    trk = [[1, 10, *A, 1], [1, 11, *B, 1]]
    assert (_ev(gt, trk, 1, "MOT15")["TP"], _ev(gt, trk, 1, "MOT15")["FP"]) == (2, 0)
    assert (_ev(gt, trk, 1)["TP"], _ev(gt, trk, 1)["FP"]) == (1, 0)


def test_combined_sums_counts_and_motp_in_order():
    gt, frames = sequence(np.random.default_rng(1), 30)
    a = mot_ref.evaluate("a", gt, _trk(frames), 30)
    b = mot_ref.evaluate("b", gt[:40], _trk(frames), 30)
    c = mot_ref.combine([a, b])
    assert c["TP"] == a["TP"] + b["TP"] and c["MOTP_sum"] == a["MOTP_sum"] + b["MOTP_sum"]
    assert c["MOTA"] == (c["TP"] - c["FP"] - c["IDSW"]) / max(1, c["TP"] + c["FN"])


# -- inputs and refusals ----------------------------------------------------------------------------------------------------
SEQINFO = """[Sequence]
name=MOT17-02-FRCNN
imDir=img1
frameRate=30
seqLength=600
imWidth=1920
imHeight=1080
imExt=.jpg
"""


def test_seqinfo_and_both_gt_layouts(tmp_path):
    from k210_yolo_framework_b200.evaluate import load_mot_gt, read_seqinfo
    (tmp_path / "seqinfo.ini").write_text(SEQINFO)
    assert read_seqinfo(str(tmp_path)) == dict(name="MOT17-02-FRCNN", imDir="img1", imExt=".jpg", frameRate=30, seqLength=600,
                                               imWidth=1920, imHeight=1080)
    (tmp_path / "gt17.txt").write_text("1,1,912,484,97,109,0,7,1\n2,3,1338.5,418,167,379,1,1,0.86\n")
    assert load_mot_gt(str(tmp_path / "gt17.txt")).tolist() == [[1, 1, 912, 484, 97, 109, 0, 7], [2, 3, 1338.5, 418, 167, 379, 1, 1]]
    (tmp_path / "gt15.txt").write_text("1,1,912,484,97,109,1,-1,-1,-1\n")
    assert load_mot_gt(str(tmp_path / "gt15.txt"), "MOT15").tolist() == [[1, 1, 912, 484, 97, 109, 1, 1]]
    with pytest.raises(ValueError):
        load_mot_gt(str(tmp_path / "gt15.txt"), "MOT17")
    (tmp_path / "bad").mkdir()
    (tmp_path / "bad" / "seqinfo.ini").write_text(SEQINFO.replace("seqLength=600\n", ""))
    with pytest.raises(ValueError, match="seqLength"):
        read_seqinfo(str(tmp_path / "bad"))


@pytest.mark.parametrize("gt,trk,match", [
    ([[0, 1, *A, 1, 1]], [], "gt frame 0 is outside 1..5"),
    ([[6, 1, *A, 1, 1]], [], "gt frame 6 is outside 1..5"),
    ([[2, 1, *A, 1, 1], [2, 1, *A, 1, 1]], [], "gt id 1 appears twice in frame 2"),
    ([[2, 1, *A, 1, 14]], [], "gt class 14 in frame 2 is outside 1..13"),
    ([], [[7, 3, *A, 1]], "tracker frame 7 is outside 1..5"),
    ([], [[3, 3, *A, 1], [3, 3, *A, 1]], "tracker id 3 appears twice in frame 3"),
])
def test_refusals(gt, trk, match):
    from k210_yolo_framework_b200.evaluate import check_mot_gt
    gt, trk = np.array(gt, np.float64).reshape(-1, 8), np.array(trk, np.float64).reshape(-1, 7)
    with pytest.raises(ValueError, match="seq: " + match):
        mot_ref.evaluate("seq", gt, trk, 5)
    if len(gt):
        with pytest.raises(ValueError, match="seq: " + match):
            check_mot_gt("seq", gt, 5, "MOT17")
    if "class" in match:        # MOT15 rows have no class
        mot_ref.check_rows("seq", gt, trk, 5, "MOT15")
        check_mot_gt("seq", gt, 5, "MOT15")
