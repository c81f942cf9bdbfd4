"""MotEval's HOTA on the GPU equals oracle/mot_hota_ref.py exactly (counts equal, every float field equal) on seeded
sequences, several sequences at once, device and pinned host blocks given in shuffled order, an empty tracker, a dense
MOT20-like sequence; and evaluate_mot.py's HOTA of its written results."""
import numpy as np
import pytest
import torch

from mot_sequences import blocks, sequence
from oracle import mot_hota_ref, mot_ref
from test_gpu_mot import _args, _frames_of, _mot_sequence, _read_results
from test_mot_ref import _chain

pytestmark = pytest.mark.gpu
PERSON = 14


def _run(benchmark, seqs, device_views=True, split=37, seed=0, K=100):
    """MotEval's result over seqs [(name, gt, frames, L)], frames fed in shuffled batches; and the restatement's HOTA."""
    from k210_yolo_framework_b200.evaluate import MotEval
    rng = np.random.default_rng(seed)
    ev = MotEval(benchmark, device=0)
    ref = {}
    for name, gt, frames, L in seqs:
        ev.add_sequence(name, gt, L)
    for name, gt, frames, L in seqs:
        ids, boxes, dets, counts = blocks(frames, K=K, rng=rng)
        trk = mot_ref.tracker_rows(range(L), ids, boxes, dets, counts, PERSON)
        ref[name] = mot_hota_ref.evaluate_hota(name, gt, trk, L, benchmark)
        starts = list(range(0, L, split))
        rng.shuffle(starts)
        for a in starts:
            sl = slice(a, a + split)
            blk = [torch.from_numpy(np.ascontiguousarray(x[sl])) for x in (ids, boxes, dets, counts)]
            blk = [b.cuda() for b in blk] if device_views else [b.pin_memory() for b in blk]
            ev.update(name, range(a, min(a + split, L)), *blk, PERSON)
    return ev.result(), ref


def _check(res, ref):
    assert set(res["hota"]["sequences"]) == set(ref)
    for name, r in ref.items():
        assert res["hota"]["sequences"][name] == r, name
    assert res["hota"]["combined"] == mot_hota_ref.combine_hota(list(ref.values()))


@pytest.mark.parametrize("benchmark,L,n_ped,seed", [("MOT17", 200, 21, 0), ("MOT20", 150, 40, 1), ("MOT15", 120, 15, 2),
                                                    ("MOT17", 400, 45, 3)])
def test_equals_the_restatement_on_seeded_sequences(benchmark, L, n_ped, seed):
    gt, frames = sequence(np.random.default_rng(seed), L, n_ped=n_ped, ambiguous=0.4, benchmark=benchmark)
    res, ref = _run(benchmark, [("s", gt, frames, L)], seed=seed)
    _check(res, ref)
    h = ref["s"]
    assert 0 < h["HOTA"][-1] < h["HOTA"][0] < 1 and h["AssA"][0] < 1


def test_several_sequences_empty_frames_ties_and_an_empty_tracker_from_host_and_device_blocks():
    seqs = []
    for k in range(3):
        gt, frames = sequence(np.random.default_rng(20 + k), 90, ambiguous=0.5)
        for f in range(10 + k, 20 + k):
            frames[f] = []
        seqs.append((f"seq{k}", gt[gt[:, 0] % 17 != 0], frames, 90))
    gt, trk = _chain(60)
    seqs.append(("chain", gt, _frames_of(trk, 60), 60))
    seqs.append(("empty", gt, [[] for _ in range(60)], 60))
    for device_views in (False, True):
        res, ref = _run("MOT17", seqs, device_views=device_views, split=8)
        _check(res, ref)
    e = res["hota"]["sequences"]["empty"]
    assert e["HOTA_FN"] == [len(gt)] * 19 and e["LocA"] == [1.0] * 19 and e["HOTA"] == [0.0] * 19
    # "sequences" and "combined" stay CLEAR and Identity
    assert set(res) == {"sequences", "combined", "rounds", "solved", "hota"} and "HOTA" not in res["combined"]


def test_a_dense_mot20_like_sequence():
    gt, frames = sequence(np.random.default_rng(2020), 12, n_ped=260, n_other=20, ambiguous=0.3, benchmark="MOT20",
                          life=(12, 12))
    assert min(len(f) for f in frames) >= 200
    res, ref = _run("MOT20", [("dense", gt, frames, 12)], K=320)
    _check(res, ref)


def test_evaluate_mot_hota_end_to_end(tmp_path):
    import evaluate_mot
    d1 = _mot_sequence(tmp_path / "train", "PEOPLE-01", 9)
    d2 = _mot_sequence(tmp_path / "train", "PEOPLE-02", 6)
    out = tmp_path / "res"
    res = evaluate_mot.evaluate(_args(tmp_path, [tmp_path / "train"], results=out))
    refs = []
    for d, name, L in ((d1, "PEOPLE-01", 9), (d2, "PEOPLE-02", 6)):
        trk = _read_results(out / f"{name}.txt")
        gt = np.loadtxt(d / "gt" / "gt.txt", delimiter=",", ndmin=2)[:, :8]
        refs.append(mot_hota_ref.evaluate_hota(name, gt, trk, L))
        assert res["hota"]["sequences"][name] == refs[-1]
    assert res["hota"]["combined"] == mot_hota_ref.combine_hota(refs)
    text = evaluate_mot.report(res)
    assert "HOTALocA(0)" in text and text.count("COMBINED") == 2
    assert evaluate_mot.to_json(res)["hota"] == res["hota"]
    # the results as the gt: 1.0 everywhere
    trk = _read_results(out / "PEOPLE-01.txt")
    (d1 / "gt" / "gt.txt").write_text("".join(f"{int(r[0])},{int(r[1])},{r[2]!r},{r[3]!r},{r[4]!r},{r[5]!r},1,1,1\n"
                                              for r in trk.tolist()))
    h = evaluate_mot.evaluate(_args(tmp_path, [d1]))["hota"]["sequences"]["PEOPLE-01"]
    for k in ("HOTA", "DetA", "AssA", "LocA", "OWTA"):
        assert h[k] == [1.0] * 19, k
    assert h["HOTA(0)"] == h["LocA(0)"] == h["HOTALocA(0)"] == 1.0
