"""Seeded MOTChallenge-like sequences for the tracking-evaluation tests and scripts/bench_mot_eval.py: gt rows and the
tracker's record blocks, as ``DetectionPipeline.collect`` / ``tracks`` give them."""
import numpy as np

MOT17_TRAIN_LENGTHS = (600, 1050, 837, 525, 654, 900, 750)


def sequence(rng, L, n_ped=21, n_other=5, ambiguous=0.2, benchmark="MOT17", life=None):
    """(gt float64 [n, 8], frames): pedestrians walking across a 1920 x 1080 view, some crossing in pairs, plus zero-marked
    and distractor rows; frames[f] lists the tracker records (id, (ymin, xmin, ymax, xmax), score) of frame f + 1, made from
    the gt with jitter, misses, false positives, ghost boxes beside a pedestrian, id switches and swapped ids where two
    pedestrians cross.  Each object is in view for life = (least, most) frames, by default L // 3 to L."""
    lo, hi = life or (max(2, L // 3), L)
    objs = []
    for i in range(n_ped + n_other):
        life = int(rng.integers(lo, hi + 1))
        start = int(rng.integers(1, L - life + 2))
        cls = 1 if i < n_ped else int(rng.choice([2, 7, 8, 12, 6, 3]))
        objs.append(dict(id=i + 1, p=rng.random(2) * [1800, 900], v=rng.normal(size=2) * 2.5, wh=[30 + rng.random() * 50,
                    90 + rng.random() * 120], cls=cls if benchmark != "MOT15" else 1, conf=0 if rng.random() < 0.08 else 1,
                    start=start, life=life))
    for a in range(0, min(n_ped, 6), 2):        # crossing pairs: b walks through a's path
        objs[a + 1].update(p=objs[a]["p"] + [200, 0], v=objs[a]["v"] - [200 / max(1, L // 2), 0], start=objs[a]["start"],
                           life=objs[a]["life"], wh=objs[a]["wh"])
    track = {o["id"]: 1000 + o["id"] for o in objs}
    nxt = 5000
    gt, frames = [], []
    for f in range(1, L + 1):
        recs = []
        for o in objs:
            if not o["start"] <= f < o["start"] + o["life"]:
                continue
            x, y = o["p"] + o["v"] * (f - o["start"])
            w, h = o["wh"]
            gt.append([f, o["id"], round(x), round(y), round(w), round(h), o["conf"], o["cls"]])
            if rng.random() < 0.08:
                continue
            if rng.random() < 0.004:
                track[o["id"]] = nxt
                nxt += 1
            j = rng.normal(size=4) * (6.0 if rng.random() < ambiguous else 1.5)
            recs.append([track[o["id"]], x + j[0], y + j[1], w + j[2], h + j[3]])
            if rng.random() < ambiguous * 0.3:
                recs.append([nxt, x + j[1] * 2, y + j[0] * 2, w, h])
                nxt += 1
        for a in range(0, min(n_ped, 6), 2):    # swapped ids while a crossing pair overlaps
            ia = [k for k, r in enumerate(recs) if r[0] == track[a + 1]]
            ib = [k for k, r in enumerate(recs) if r[0] == track[a + 2]]
            if ia and ib and rng.random() < 0.3:
                recs[ia[0]][0], recs[ib[0]][0] = recs[ib[0]][0], recs[ia[0]][0]
        for _ in range(int(rng.integers(0, 3))):
            recs.append([nxt, rng.random() * 1800, rng.random() * 900, 40.0, 110.0])
            nxt += 1
        rng.shuffle(recs)
        frames.append([(int(r[0]), (r[2], r[1], r[2] + r[4], r[1] + r[3]), float(rng.random())) for r in recs])
    return np.array(gt, np.float64).reshape(-1, 8), frames


def blocks(frames, C=20, K=100, person=14, rng=None):
    """(ids int32 [F, C, K], boxes float32 [F, C, K, 4], dets int32 [F, C, K, 6], counts int32 [F, C]) of the frames' records
    as person records, beside untracked person records (id -1) and records of another class."""
    F = len(frames)
    ids = np.full((F, C, K), -1, np.int32)
    boxes = np.zeros((F, C, K, 4), np.float32)
    dets = np.zeros((F, C, K, 6), np.int32)
    counts = np.zeros((F, C), np.int32)
    rng = rng or np.random.default_rng(0)
    for f, recs in enumerate(frames):
        rows = list(recs)
        for _ in range(int(rng.integers(0, 2))):
            rows.insert(int(rng.integers(0, len(rows) + 1)), (-1, (10.0, 10.0, 60.0, 30.0), 0.1))
        rows = rows[:K]
        for k, (t, b, s) in enumerate(rows):
            ids[f, person, k] = t
            boxes[f, person, k] = b
            dets[f, person, k, :5] = np.array(list(b) + [s], np.float32).view(np.int32)
        counts[f, person] = len(rows)
        other = (person + 1) % C
        ids[f, other, 0], boxes[f, other, 0], counts[f, other] = 7, (5, 5, 90, 90), 1
    return ids, boxes, dets, counts
