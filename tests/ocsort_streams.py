"""Seeded record streams for the OC-SORT tests: objects per class that turn, cross one another, vanish for 1 to max_age + 2
frames and come back off the path they were on, score spans in the low band (0.1, det_thresh), identical duplicates
(assignment ties), scores exactly at det_thresh, zero-area and non-finite records."""
import numpy as np


def stream(rng, C, K, n_frames, n_obj=12, size=600.0, max_age=30, det_thresh=0.6):
    """[n_frames] of (boxes float32 [C, K, 4] (ymin, xmin, ymax, xmax), counts int32 [C], scores float32 [C, K])."""
    objs = []
    for _ in range(C):
        cls = []
        for _ in range(int(rng.integers(0, n_obj + 1))):
            cls.append(dict(start=int(rng.integers(0, n_frames)), life=int(rng.integers(2, n_frames)), p=rng.random(2) * size,
                            v=rng.normal(size=2) * 5, turn=float(rng.normal() * 0.15), wh=12 + rng.random(2) * 60,
                            occ=int(rng.integers(0, n_frames)), occ_len=int(rng.integers(1, max_age + 3)),
                            jump=rng.normal(size=2) * 12, low=int(rng.integers(0, n_frames)), low_len=int(rng.integers(1, 6)),
                            base=float(rng.uniform(det_thresh - 0.05, 0.98))))
        objs.append(cls)
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for c in range(C):
            recs = []
            for o in objs[c]:
                age = f - o["start"]
                if not 0 <= age < o["life"] or o["occ"] <= f < o["occ"] + o["occ_len"] or rng.random() < 0.05:
                    continue
                a = o["turn"] * age                     # the velocity turns by `turn` radians a frame
                v = np.array([o["v"][0] * np.cos(a) - o["v"][1] * np.sin(a), o["v"][0] * np.sin(a) + o["v"][1] * np.cos(a)])
                ctr = o["p"] + v * age + rng.normal(size=2) * 1.5
                if f >= o["occ"] + o["occ_len"]:
                    ctr = ctr + o["jump"]               # back off the path it was on
                box = [ctr[1] - o["wh"][1] / 2, ctr[0] - o["wh"][0] / 2, ctr[1] + o["wh"][1] / 2, ctr[0] + o["wh"][0] / 2]
                s = o["base"] + rng.normal() * 0.05
                if o["low"] <= f < o["low"] + o["low_len"]:
                    s = rng.uniform(0.12, det_thresh - 0.02)
                if rng.random() < 0.04:
                    s = det_thresh
                recs.append(box + [min(max(s, 0.0), 1.0)])
            if recs and rng.random() < 0.25:
                recs.append(list(recs[int(rng.integers(0, len(recs)))]))
            if rng.random() < 0.3:
                y, x = rng.random(2) * size
                recs.append([y, x, y + 20, x + 30, float(rng.uniform(0.0, 0.3))])
            if rng.random() < 0.08:
                recs.append([3.0, 3.0, 3.0, 40.0, 0.9])
            if rng.random() < 0.03:
                recs.append([0.0, 0.0, 10.0, np.inf, 0.9])
            if rng.random() < 0.02:
                recs.append([np.nan, 0.0, 10.0, 10.0, 0.9])
            rng.shuffle(recs)
            recs = recs[:K]
            if recs:
                arr = np.array(recs, np.float64)
                boxes[c, :len(recs)] = arr[:, :4].astype(np.float32)
                scores[c, :len(recs)] = arr[:, 4].astype(np.float32)
            counts[c] = len(recs)
        out.append((boxes, counts, scores))
    return out


def crowded(C, K, n_frames):
    """Class 0 fills its track bound: K new boxes in each frame, overlapping nothing of before, each seen once and then
    kept until max_age removes it; the last class holds one slowly growing box."""
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for i in range(K):
            y, x = 40.0 * i, 100.0 + 40.0 * f
            boxes[0, i] = [y, x, y + 10, x + 10]
            scores[0, i] = 0.9
        counts[0] = K
        counts[C - 1] = 1
        boxes[C - 1, 0] = [5, 5, 50, 50 + f]
        scores[C - 1, 0] = 0.8
        out.append((boxes, counts, scores))
    return out
