"""Seeded record streams for the ByteTrack tests: objects per class that move, cross, leave and come back, with scores in
both bands (an occlusion drops an object's score into the low band for a few frames), scores at exactly track_thresh and
between track_thresh and det_thresh, identical duplicates (assignment ties), low-score clutter, zero-area and non-finite
records."""
import numpy as np


def stream(rng, C, K, n_frames, n_obj=12, size=600.0, track_thresh=0.5):
    """[n_frames] of (boxes float32 [C, K, 4] (ymin, xmin, ymax, xmax), counts int32 [C], scores float32 [C, K])."""
    objs = []
    for _ in range(C):
        objs.append([dict(start=int(rng.integers(0, n_frames)), life=int(rng.integers(2, n_frames)), p=rng.random(2) * size,
                          v=rng.normal(size=2) * 6, wh=10 + rng.random(2) * 70, occ=int(rng.integers(0, n_frames)),
                          occ_len=int(rng.integers(1, 6)), base=float(rng.uniform(0.55, 0.98)))
                     for _ in range(int(rng.integers(0, n_obj + 1)))])
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for c in range(C):
            recs = []
            for o in objs[c]:
                if not o["start"] <= f < o["start"] + o["life"] or rng.random() < 0.08:
                    continue
                ctr = o["p"] + o["v"] * (f - o["start"]) + rng.normal(size=2) * 1.5
                box = [ctr[1] - o["wh"][1] / 2, ctr[0] - o["wh"][0] / 2, ctr[1] + o["wh"][1] / 2, ctr[0] + o["wh"][0] / 2]
                s = o["base"] + rng.normal() * 0.05
                if o["occ"] <= f < o["occ"] + o["occ_len"]:
                    s = rng.uniform(0.12, 0.45)
                r = rng.random()
                if r < 0.04:
                    s = track_thresh
                elif r < 0.1:
                    s = track_thresh + 0.05
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
            rng.shuffle(recs)
            recs = recs[:K]
            if recs:
                a = np.array(recs, np.float64)
                boxes[c, :len(recs)] = a[:, :4].astype(np.float32)
                scores[c, :len(recs)] = a[:, 4].astype(np.float32)
            counts[c] = len(recs)
        out.append((boxes, counts, scores))
    return out


def crowded(C, K, n_frames):
    """Class 0 fills its track bound: K new high-score boxes in each frame, overlapping nothing of before, so each frame's
    records are born, confirmed the next frame by the record that follows them and then lost, until track_buffer removes
    them; the last class holds one slowly growing box."""
    out = []
    for f in range(n_frames):
        boxes = np.zeros((C, K, 4), np.float32)
        scores = np.zeros((C, K), np.float32)
        counts = np.zeros(C, np.int32)
        for i in range(K):
            y, x = 40.0 * i, 100.0 + 40.0 * (f // 2)
            boxes[0, i] = [y, x, y + 10, x + 10]
            scores[0, i] = 0.9
        counts[0] = K
        counts[C - 1] = 1
        boxes[C - 1, 0] = [5, 5, 50, 50 + f]
        scores[C - 1, 0] = 0.8
        out.append((boxes, counts, scores))
    return out
